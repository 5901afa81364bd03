// mgf_kernels.cu -- Fourier / moment-generating-function hot path for sm_90a (H100).
//
// Replaces (paths under /root/reference/src/stochvolmodels):
//   func_a_ode_quadratic_terms, func_rhs            pricers/logsv/affine_expansion.py:67-205
//   solve_ode_for_a / solve_a_ode_grid (RK45)       pricers/logsv/affine_expansion.py:229-303, 492-529
//       -> scipy.integrate.solve_ivp(method="RK45", rtol=1e-3, atol=1e-6): scipy/integrate/_ivp/rk.py, common.py
//   compute_logsv_a_mgf_grid (log-MGF contraction)  pricers/logsv/affine_expansion.py:570-685
//   logsv_chain_pricer (LOG_RETURN)                 pricers/logsv_pricer.py:669-739
//   compute_heston_mgf_grid, heston_chain_pricer    pricers/heston_pricer.py:183-282
//   get_phi_grid, _compute_legacy_pricer_weights, vanilla_slice_pricer_with_mgf_grid   utils/mgf_pricer.py:11-34,157-221
//
// Design (DESIGN.md §4): the grid is P = 1000 independent ODE systems per maturity -- latency bound, no data reuse, no
// tensor-core shape.  One thread integrates one grid point through ALL maturities of the chain with the coefficient
// vector A in registers (the reference carries a_t0 across maturities the same way), using the exact step-size control
// law of SciPy's RK45 so that accepted steps -- and therefore prices -- match the reference to ~1e-13.  CTAs are kept
// tiny (8..64 threads) so the 1000 threads spread over as many SMs as possible and a warp waits for few slow lanes.
// A second kernel does the Simpson-weighted Fourier sums, one CTA per strike, fixed-order fp64 reduction.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <mutex>
#include <type_traits>
#include <vector>

#include "../../include/b200sv.h"
#include "common.cuh"
#include "black.cuh"
#include "fastmath64.cuh"

namespace b200sv {

struct cd {
  double re, im;
};
__host__ __device__ __forceinline__ cd mk(double re, double im = 0.0) { return cd{re, im}; }
__device__ __forceinline__ cd operator+(cd a, cd b) { return cd{a.re + b.re, a.im + b.im}; }
__device__ __forceinline__ cd operator-(cd a, cd b) { return cd{a.re - b.re, a.im - b.im}; }
__device__ __forceinline__ cd operator-(cd a) { return cd{-a.re, -a.im}; }
__device__ __forceinline__ cd operator*(cd a, cd b) { return cd{a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re}; }
__device__ __forceinline__ cd operator*(double s, cd a) { return cd{s * a.re, s * a.im}; }
__device__ __forceinline__ cd operator*(cd a, double s) { return cd{s * a.re, s * a.im}; }
__device__ __forceinline__ double cabs2(cd a) { return a.re * a.re + a.im * a.im; }
__device__ __forceinline__ double cabs_(cd a) { return hypot(a.re, a.im); }
// Smith's division (what numpy uses for complex128)
__device__ __forceinline__ cd operator/(cd a, cd b) {
  if (fabs(b.re) >= fabs(b.im)) {
    const double r = b.im / b.re, d = b.re + b.im * r;
    return cd{(a.re + a.im * r) / d, (a.im - a.re * r) / d};
  }
  const double r = b.re / b.im, d = b.re * r + b.im;
  return cd{(a.re * r + a.im) / d, (a.im * r - a.re) / d};
}
__device__ __forceinline__ cd sqrt_(cd z) {   // principal branch
  if (z.re == 0.0 && z.im == 0.0) return cd{0.0, z.im};
  const double t = sqrt(0.5 * (fabs(z.re) + hypot(z.re, z.im)));
  if (z.re >= 0.0) return cd{t, z.im / (2.0 * t)};
  return cd{fabs(z.im) / (2.0 * t), copysign(t, z.im)};
}
__device__ __forceinline__ cd exp_(cd z) {
  double s, c;
  sincos(z.im, &s, &c);
  const double e = exp(z.re);
  return cd{e * c, e * s};
}
__device__ __forceinline__ cd log_(cd z) { return cd{log(hypot(z.re, z.im)), atan2(z.im, z.re)}; }
// exp_ with C99 cexp's exp(x ± 0i) = exp(x) ± 0i, which is numpy's: the summand of the strike sums at Im = 0 (grid point 0) whose exponent
// overflows is then +inf, kept by np.nansum, instead of inf * sin(0) = NaN, skipped.  Used by the strike-sum kernels only; wherever exp_(z)
// is finite the two agree bit for bit.
__device__ __forceinline__ cd cexp_(cd z) {
  const cd e = exp_(z);
  return cd{e.re, z.im == 0.0 ? z.im : e.im};
}

// --------------------------------------------------------------------------------------------------------------------
// LogSV affine expansion: per-grid-point coefficients of A' = A^T M A + L A + H (sparse, hand-expanded)
// --------------------------------------------------------------------------------------------------------------------
struct LogsvModel {   // phi-independent reals, built on the host: affine_expansion.py:121-135
  double theta, th2, v2, qv, qv2, lam, k2p, kp, beta_eta, eta2;
  int spot;
};

static LogsvModel make_model(const b200sv_logsv_params& p, double eta, bool spot) {
  LogsvModel m;
  m.theta = p.theta;
  m.th2 = p.theta * p.theta;
  m.v2 = p.beta * p.beta + p.volvol * p.volvol;
  m.qv = p.theta * m.v2;
  m.qv2 = m.th2 * m.v2;
  m.eta2 = eta * eta;
  if (spot) {
    m.lam = 0.0;
    m.k2p = p.kappa2;
    m.kp = p.kappa1 + p.kappa2 * p.theta;
  } else {
    m.lam = p.beta * m.th2 * eta;
    m.k2p = p.kappa2 - p.beta * eta;
    m.kp = p.kappa1 + p.kappa2 * p.theta - 2 * p.beta * p.theta * eta;
  }
  m.beta_eta = p.beta * eta;
  m.spot = spot ? 1 : 0;
  return m;
}

struct Coef {   // the phi/psi-dependent entries of L and H (affine_expansion.py:166-183)
  cd l01, l11, l12, l21, l22, l23, l32, l33, l34, l43, l44, h0, h1, h2;
};

__device__ __forceinline__ Coef make_coef(const LogsvModel& m, cd phi, cd psi) {
  Coef c;
  const cd b = m.beta_eta * phi;
  c.l01 = mk(m.lam) - m.th2 * b;
  c.l11 = mk(-m.kp) - (2.0 * m.theta) * b;
  c.l12 = 2.0 * (mk(m.lam + m.qv) - m.th2 * b);
  c.l21 = mk(-m.k2p) - b;
  c.l22 = mk(m.v2 - 2.0 * m.kp) - (4.0 * m.theta) * b;
  c.l23 = 3.0 * (mk(2.0 * m.qv) - m.th2 * b);
  c.l32 = -2.0 * (mk(m.k2p) + b);
  c.l33 = 3.0 * (mk(m.v2 - m.kp) - (2.0 * m.theta) * b);
  c.l34 = 4.0 * (mk(3.0 * m.qv) - m.th2 * b);
  c.l43 = -3.0 * (mk(m.k2p) + b);
  c.l44 = 2.0 * (mk(m.v2 - 2.0 * m.kp) - (4.0 * m.theta) * b);
  const cd r = m.spot ? phi * (phi + mk(1.0)) - 2.0 * psi : phi * (phi - mk(1.0)) - 2.0 * psi;
  c.h0 = (0.5 * m.th2 * m.eta2) * r;
  c.h1 = (m.theta * m.eta2) * r;
  c.h2 = (0.5 * m.eta2) * r;
  return c;
}

// The 14 phi/psi-dependent coefficients of one thread, parked in shared memory ([coef][thread]) like the RK stages: the kernel is
// latency-bound, so register space is better spent on independent in-flight products than on long-lived constants.
template <int TPB>
struct CoefView {
  const cd* base;
  __device__ __forceinline__ cd at(int i) const { return base[i * TPB]; }
};
template <int TPB>
__device__ __forceinline__ void store_coef(cd* base, const Coef& c) {
  const cd v[14] = {c.l01, c.l11, c.l12, c.l21, c.l22, c.l23, c.l32, c.l33, c.l34, c.l43, c.l44, c.h0, c.h1, c.h2};
#pragma unroll
  for (int i = 0; i < 14; ++i) base[i * TPB] = v[i];
}

template <int N, int TPB>
__device__ __forceinline__ void rhs(const cd (&A)[N], const LogsvModel& m, const CoefView<TPB>& cv, cd (&out)[N]) {
  struct {
    cd l01, l11, l12, l21, l22, l23, l32, l33, l34, l43, l44, h0, h1, h2;
  } c;
  c.l01 = cv.at(0); c.l11 = cv.at(1); c.l12 = cv.at(2); c.l21 = cv.at(3); c.l22 = cv.at(4); c.h0 = cv.at(11); c.h1 = cv.at(12); c.h2 = cv.at(13);
  if constexpr (N == 5) {
    c.l23 = cv.at(5); c.l32 = cv.at(6); c.l33 = cv.at(7); c.l34 = cv.at(8); c.l43 = cv.at(9); c.l44 = cv.at(10);
  }
  const double v2 = m.v2, qv = m.qv, qv2 = m.qv2;
  const cd a1 = A[1], a2 = A[2];
  const cd a11 = a1 * a1, a12 = a1 * a2, a22 = a2 * a2;
  if constexpr (N == 5) {
    const cd a3 = A[3], a4 = A[4];
    const cd a13 = a1 * a3, a14 = a1 * a4, a23 = a2 * a3, a24 = a2 * a4, a33 = a3 * a3;
    out[0] = (0.5 * qv2) * a11 + c.l01 * a1 + qv2 * a2 + c.h0;
    out[1] = qv * a11 + (2.0 * qv2) * a12 + c.l11 * a1 + c.l12 * a2 + (3.0 * qv2) * a3 + c.h1;
    out[2] = (0.5 * v2) * a11 + (2.0 * qv2) * a22 + (4.0 * qv) * a12 + (3.0 * qv2) * a13 + c.l21 * a1 + c.l22 * a2 + c.l23 * a3 +
             (6.0 * qv2) * a4 + c.h2;
    out[3] = (4.0 * qv) * a22 + (2.0 * v2) * a12 + (6.0 * qv) * a13 + (4.0 * qv2) * a14 + (6.0 * qv2) * a23 + c.l32 * a2 +
             c.l33 * a3 + c.l34 * a4;
    out[4] = (2.0 * v2) * a22 + (4.5 * qv2) * a33 + (3.0 * v2) * a13 + (8.0 * qv) * a14 + (12.0 * qv) * a23 + (8.0 * qv2) * a24 +
             c.l43 * a3 + c.l44 * a4;
  } else {
    out[0] = (0.5 * qv2) * a11 + c.l01 * a1 + qv2 * a2 + c.h0;
    out[1] = qv * a11 + (2.0 * qv2) * a12 + c.l11 * a1 + c.l12 * a2 + c.h1;
    out[2] = (0.5 * v2) * a11 + (2.0 * qv2) * a22 + (4.0 * qv) * a12 + c.l21 * a1 + c.l22 * a2 + c.h2;
  }
}

// --------------------------------------------------------------------------------------------------------------------
// SciPy RK45 clone (scipy/integrate/_ivp/rk.py:111-170 step loop, :14-69 stages, :538-552 tableau;
//                   scipy/integrate/_ivp/common.py:63-65 norm, :109-134 select_initial_step)
// --------------------------------------------------------------------------------------------------------------------
__constant__ double c_A[6][5] = {{0, 0, 0, 0, 0},
                                 {1.0 / 5, 0, 0, 0, 0},
                                 {3.0 / 40, 9.0 / 40, 0, 0, 0},
                                 {44.0 / 45, -56.0 / 15, 32.0 / 9, 0, 0},
                                 {19372.0 / 6561, -25360.0 / 2187, 64448.0 / 6561, -212.0 / 729, 0},
                                 {9017.0 / 3168, -355.0 / 33, 46732.0 / 5247, 49.0 / 176, -5103.0 / 18656}};   // Dormand-Prince A (rk.py:542-549)
constexpr double kRtol = 1e-3, kAtol = 1e-6;   // solve_ivp defaults, affine_expansion.py:300-301 passes none

// Step-size control arithmetic of the RK45 clone (error scale, RMS norm): MUFU-seeded reciprocal / square root with Newton refinement
// (<= 2 ulp, fastmath64.cuh) instead of the IEEE sequences with their slow-path branches -- these sit on the dependent chain of every
// step attempt.  Moduli below 1e-145 count as 0 (the scale is atol + |a| rtol with atol = 1e-6: identical result).
__device__ __forceinline__ double ctrl_sqrt(double s) { return s < 1e-290 ? 0.0 : fast_sqrt(s); }
__device__ __forceinline__ double ctrl_rcp(double x) { return fast_div(1.0, x); }     // x >= atol
// RMS norm of v / scale over complex moduli (scipy/integrate/_ivp/common.py:63-65); inv_scale = 1 / scale.
template <int N>
__device__ __forceinline__ double rms_scaled(const cd (&v)[N], const double (&inv_scale)[N]) {
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    const double re = v[k].re * inv_scale[k], im = v[k].im * inv_scale[k];
    s += re * re + im * im;
  }
  return ctrl_sqrt(s) * (N == 5 ? 0.44721359549995793 : 0.57735026918962576);   // / sqrt(N)
}
__device__ __forceinline__ double cmod(cd a) { return ctrl_sqrt(a.re * a.re + a.im * a.im); }   // |a| (no overflow risk for these magnitudes)
// e^(-1/5), e > 0, for the step-size factor 0.9 e^(-1/5) clipped to [0.2, 10]: SFU single-precision seed + two Newton steps on x^-5 = e
// (x <- x (1.2 - 0.2 e x^5), quadratic: 1e-6 -> 3e-12 -> 1 ulp) instead of exp(-0.2 log e).  Outside [1e-30, 1e30] the clipped factor
// does not depend on e, so e is clamped for the float seed; NaN propagates (fmax(0.2, NaN) = 0.2 as before).
__device__ __forceinline__ double pow_m02(double e) {
  const double ec = e != e ? e : fmin(fmax(e, 1e-30), 1e30);
  double x = (double)__powf((float)ec, -0.2f);
  const double c = 0.2 * ec;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const double x2 = x * x;
    x = x * fma(-c, x2 * x2 * x, 1.2);
  }
  return x;
}

// Stage storage of one thread in shared memory: K[stage][component][thread] (16-byte elements, conflict-free across threads).
// Keeping the 7 x N complex stages out of the register file leaves ptxas room to schedule the independent products of the
// right-hand side in parallel: the kernel is latency-bound (one warp per SM), so ILP is what matters.
template <int N, int TPB>
struct StageStore {
  cd* base;
  __device__ __forceinline__ cd& at(int stage, int k) { return base[(stage * N + k) * TPB]; }
};

// No tangent: the default of rk45_generic, every hook call compiles away.
struct NoTangent {};

// returns 0 ok, 1 step size underflow (SciPy: TOO_SMALL_STEP -> solver fails, reference keeps the last accepted state)
// Rhs: functor ``void operator()(const cd (&A)[N], cd (&out)[N]) const`` -- the LogSV coefficient ODEs (LogsvRhsFn) or the Hawkes Riccati
// system (HawkesRhsFn); the control law does not depend on it.
// Tan (optional, LogsvTangentHook): a forward-mode derivative stepped on the SAME attempts -- it sees every stage input, the step size
// and the acceptance, and never feeds back into the error norm, so the mesh is the primal's.
template <int N, int TPB, typename Rhs, typename Tan = NoTangent>
__device__ int rk45_generic(cd (&y)[N], double T, const Rhs& rhs_fn, StageStore<N, TPB> K, int* nfev_out, Tan* tan = nullptr) {
  constexpr bool kTan = !std::is_same<Tan, NoTangent>::value;
  // stage coefficients: c_A in constant memory (indexed by the non-unrolled stage loop)
  constexpr double B[6] = {35.0 / 384, 0, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84};
  constexpr double E[7] = {-71.0 / 57600, 0, 71.0 / 16695, -71.0 / 1920, 17253.0 / 339200, -22.0 / 525, 1.0 / 40};

  cd f[N];                       // f(t, y): registers during the initial-step selection, then stage 0 of the shared-memory store
  rhs_fn(y, f);
  int nfev = 1;
  double inv_scale[N];
  // ---- select_initial_step (scipy/integrate/_ivp/common.py:109-134)
  double h_abs;
  {
#pragma unroll
    for (int k = 0; k < N; ++k) inv_scale[k] = ctrl_rcp(kAtol + cmod(y[k]) * kRtol);
    const double d0 = rms_scaled<N>(y, inv_scale), d1 = rms_scaled<N>(f, inv_scale);
    double h0 = (d0 < 1e-5 || d1 < 1e-5) ? 1e-6 : 0.01 * d0 / d1;
    h0 = fmin(h0, T);
    cd y1[N], f1[N];
#pragma unroll
    for (int k = 0; k < N; ++k) y1[k] = y[k] + h0 * f[k];
    rhs_fn(y1, f1);
    ++nfev;
#pragma unroll
    for (int k = 0; k < N; ++k) f1[k] = f1[k] - f[k];
    const double d2 = rms_scaled<N>(f1, inv_scale) / h0;
    const double h1 = (d1 <= 1e-15 && d2 <= 1e-15) ? fmax(1e-6, h0 * 1e-3) : exp(0.2 * log(0.01 / fmax(d1, d2)));
    h_abs = fmin(fmin(100.0 * h0, h1), T);
  }
  double t = 0.0;
  int status = 0;
#pragma unroll
  for (int k = 0; k < N; ++k) K.at(0, k) = f[k];
  if constexpr (kTan) tan->start(y);
  // ONE loop over step ATTEMPTS (SciPy nests "while not accepted" inside the step loop): a lane that rejects an attempt simply goes round
  // again with the lanes that accepted theirs, so a warp runs max-over-lanes of the TOTAL attempts instead of the sum over steps of
  // the per-step maximum.  Same arithmetic per point.
  bool rejected = false;
  for (int guard = 0; t < T && guard < 400000; ++guard) {
    {
      const double min_step = 10.0 * (__longlong_as_double(__double_as_longlong(t) + 1) - t);   // 10*|nextafter(t, inf) - t|, t >= 0
      if (!rejected) {
        if (h_abs < min_step) h_abs = min_step;       // first attempt of a step (max_step = inf)
      } else if (h_abs < min_step) {
        status = 1;
        break;
      }
      double t_new = t + h_abs;
      if (t_new - T > 0.0) t_new = T;
      const double h = t_new - t;
      h_abs = fabs(h);
      cd yt[N], kn[N];
#pragma unroll 1
      for (int s = 1; s < 6; ++s) {            // rk_step (scipy/integrate/_ivp/rk.py:60-64): dy = (sum_j K_j a_sj) * h
        // not unrolled on purpose: the fully unrolled body (5 inlined right-hand sides) is ~70 KB of SASS and the single resident
        // warp per SM then stalls on instruction fetch; stages >= s still hold zeros / stale finite values and get coefficient 0
        // (skipping them with a warp-uniform trip count was measured: no gain, more spills)
#pragma unroll
        for (int k = 0; k < N; ++k) {
          cd acc = K.at(0, k) * c_A[s][0];
#pragma unroll
          for (int jj = 1; jj < 5; ++jj) acc = acc + K.at(jj, k) * c_A[s][jj];
          yt[k] = y[k] + acc * h;
        }
        if constexpr (kTan) tan->stage(s, yt, h);
        rhs_fn(yt, kn);
#pragma unroll
        for (int k = 0; k < N; ++k) K.at(s, k) = kn[k];
      }
      cd yn[N];
#pragma unroll
      for (int k = 0; k < N; ++k) {
        cd acc = K.at(0, k) * B[0];
#pragma unroll
        for (int jj = 2; jj < 6; ++jj) acc = acc + K.at(jj, k) * B[jj];      // B[1] = 0
        yn[k] = y[k] + h * acc;
      }
      rhs_fn(yn, kn);                                                   // K[6] = f(t + h, y_new)
      if constexpr (kTan) tan->last(yn, h);
      nfev += 6;
      cd err[N];
#pragma unroll
      for (int k = 0; k < N; ++k) {
        inv_scale[k] = ctrl_rcp(kAtol + fmax(cmod(y[k]), cmod(yn[k])) * kRtol);
        cd acc = K.at(0, k) * E[0];
#pragma unroll
        for (int jj = 2; jj < 6; ++jj) acc = acc + K.at(jj, k) * E[jj];      // E[1] = 0
        err[k] = (acc + kn[k] * E[6]) * h;
      }
      const double en = rms_scaled<N>(err, inv_scale);
      const bool accepted = en < 1.0;
      const double pf = en == 0.0 ? 10.0 : 0.9 * pow_m02(en);
      double factor = fmin(10.0, pf);
      if (rejected) factor = fmin(1.0, factor);
      h_abs *= accepted ? factor : fmax(0.2, pf);
      if (accepted) {
        t = t_new;
#pragma unroll
        for (int k = 0; k < N; ++k) {
          y[k] = yn[k];
          K.at(0, k) = kn[k];     // FSAL: K[6] of this step is K[0] of the next
        }
        if constexpr (kTan) tan->accept();
      }
      rejected = !accepted;
    }
  }
  if (nfev_out) *nfev_out = nfev;
  return status;
}

template <int N, int TPB>
struct LogsvRhsFn {
  const LogsvModel& m;
  const CoefView<TPB>& c;
  __device__ __forceinline__ void operator()(const cd (&A)[N], cd (&out)[N]) const { rhs<N, TPB>(A, m, c, out); }
};
template <int N, int TPB>
__device__ __forceinline__ int rk45(cd (&y)[N], double T, const LogsvModel& m, const CoefView<TPB>& c, StageStore<N, TPB> K, int* nfev_out) {
  return rk45_generic<N, TPB>(y, T, LogsvRhsFn<N, TPB>{m, c}, K, nfev_out);
}

struct ChainSpec {   // per-maturity scalars (device array of M entries)
  double dtau;
  LogsvModel model;
};

// one thread = one grid point through all M maturities.  a_io: [P][N] in (A(0)) ; a_out: [M][P][N]; log_mgf: [M][P]
// blockIdx.y = parameter set of a batch (b200sv_logsv_price_chain_batch): spec[b][M], yb[b], phi[b][P] (phi_stride = P) or one shared
// grid (phi_stride = 0), outputs [b][M][P]...
template <int N, int TPB>
__global__ void __launch_bounds__(TPB) logsv_mgf_kernel(const cd* __restrict__ phi, const cd* __restrict__ psi, int P, int M,
                                 const ChainSpec* __restrict__ spec, const cd* __restrict__ a_in, cd* __restrict__ a_out,
                                 cd* __restrict__ log_mgf, double y, int* __restrict__ status, int* __restrict__ nfev,
                                 const double* __restrict__ yb = nullptr, int phi_stride = 0, int set_major_B = 0) {
  __shared__ cd stage_smem[6 * N * TPB];
  __shared__ cd coef_smem[14 * TPB];
  // Batches (set_major_B = B > 1): the parameter set is the FASTEST thread index, so the lanes of a warp integrate the same grid point
  // for 32 neighbouring sets -- the sets of a calibration batch are perturbations of one another and take (nearly) the same adaptive
  // steps, whereas neighbouring grid points of one set do not (24 of 32 lanes active with the point-major mapping, r01 profile).
  int p = blockIdx.x * TPB + threadIdx.x;
  size_t b = blockIdx.y;
  if (set_major_B > 1) {
    const long long t = (long long)blockIdx.x * TPB + threadIdx.x;
    if (t >= (long long)set_major_B * P) return;
    b = (size_t)(t % set_major_B);
    p = (int)(t / set_major_B);
  }
  if (p >= P) return;
  if (gridDim.y > 1 || yb) {
    spec += b * M;
    phi += b * (size_t)phi_stride;
    a_out += b * (size_t)M * P * N;
    log_mgf += b * (size_t)M * P;
    if (status) status += b * (size_t)P;
    if (yb) y = yb[b];
  }
  StageStore<N, TPB> K{stage_smem + threadIdx.x};
#pragma unroll
  for (int i = 0; i < 6 * N; ++i) stage_smem[threadIdx.x + i * TPB] = mk(0.0);      // stages read with coefficient 0 must be finite
  cd A[N];
#pragma unroll
  for (int k = 0; k < N; ++k) A[k] = a_in ? a_in[(size_t)p * N + k] : mk(0.0);
  const cd ph = phi[p], ps = psi ? psi[p] : mk(0.0);
  // ys = [1, y, y^2, y^3, y^4] (affine_expansion.py:674-681)
  const double y2 = y * y;
  const double ys[5] = {1.0, y, y2, y2 * y, y2 * y2};
  int st = 0, nf = 0;
  for (int mm = 0; mm < M; ++mm) {
    const LogsvModel model = spec[mm].model;
    store_coef<TPB>(coef_smem + threadIdx.x, make_coef(model, ph, ps));
    const CoefView<TPB> c{coef_smem + threadIdx.x};
    int nfe = 0;
    st |= rk45<N, TPB>(A, spec[mm].dtau, model, c, K, &nfe);
    nf += nfe;
    cd lm = mk(0.0);
#pragma unroll
    for (int k = 0; k < N; ++k) {
      a_out[((size_t)mm * P + p) * N + k] = A[k];
      lm = lm + A[k] * ys[k];
    }
    log_mgf[(size_t)mm * P + p] = lm;
  }
  if (status) status[p] = st;
  if (nfev) nfev[p] = nf;
}

// --------------------------------------------------------------------------------------------------------------------
// Lane-parallel variant for the latency regime (one chain, P = 1000): the N components of A are spread over N lanes of a group of LPP
// lanes (8 for N = 5, 4 for N = 3), so one Runge-Kutta stage costs each lane ONE row of A'MA + LA + H (<= 6 quadratic + 4 linear terms)
// instead of all N rows -- about a third of the dependent instruction stream of the thread-per-point kernel, which is what bounds a
// single chain pricing (one resident warp per SM).  The stage vector is exchanged through shared memory (one 16-byte store, <= 5 loads,
// __syncwarp); each lane keeps its own 7 stage derivatives in registers.  Step-size control is replicated in every lane of a point from
// an error norm summed in component order, i.e. the same accepted steps as the thread-per-point kernel; all points of a warp iterate
// together (finished points idle) so the warp-level barriers stay converged.  Row k accumulates its terms in the order of rhs<>().
// --------------------------------------------------------------------------------------------------------------------
template <int N>
struct LaneRow {        // row k of the right-hand side in table form
  cd l[4];              // linear coefficients (complex; real ones carry im = 0)
  double q[6];          // quadratic coefficients (already doubled for off-diagonal pairs)
  cd h;
  int li[4], qi[6], qj[6];
  int nl, nq;
};

template <int N>
__device__ __forceinline__ LaneRow<N> make_lane_row(int k, const LogsvModel& m, cd phi, cd psi) {
  const Coef c = make_coef(m, phi, psi);
  const double v2 = m.v2, qv = m.qv, qv2 = m.qv2;
  LaneRow<N> r;
  // padding entries: coefficient 0 on a component every row already depends on (rows 0-3: A1, row 4: A3), so that a non-finite value
  // cannot enter a row through a padded term unless the row is non-finite anyway
  const int pad = k == 4 ? 3 : 1;
#pragma unroll
  for (int t = 0; t < 4; ++t) { r.l[t] = mk(0.0); r.li[t] = pad; }
#pragma unroll
  for (int t = 0; t < 6; ++t) { r.q[t] = 0.0; r.qi[t] = pad; r.qj[t] = pad; }
  r.h = mk(0.0);
  r.nl = r.nq = 0;
  auto Q = [&](double coef, int i, int j) { r.q[r.nq] = coef; r.qi[r.nq] = i; r.qj[r.nq] = j; ++r.nq; };
  auto L = [&](cd coef, int i) { r.l[r.nl] = coef; r.li[r.nl] = i; ++r.nl; };
  // same term order as rhs<>() above (affine_expansion.py:139-183)
  if (k == 0) {
    Q(0.5 * qv2, 1, 1); L(c.l01, 1); L(mk(qv2), 2); r.h = c.h0;
  } else if (k == 1) {
    Q(qv, 1, 1); Q(2.0 * qv2, 1, 2); L(c.l11, 1); L(c.l12, 2);
    if (N == 5) L(mk(3.0 * qv2), 3);
    r.h = c.h1;
  } else if (k == 2) {
    Q(0.5 * v2, 1, 1); Q(2.0 * qv2, 2, 2); Q(4.0 * qv, 1, 2);
    if (N == 5) Q(3.0 * qv2, 1, 3);
    L(c.l21, 1); L(c.l22, 2);
    if (N == 5) { L(c.l23, 3); L(mk(6.0 * qv2), 4); }
    r.h = c.h2;
  } else if (k == 3) {
    Q(4.0 * qv, 2, 2); Q(2.0 * v2, 1, 2); Q(6.0 * qv, 1, 3); Q(4.0 * qv2, 1, 4); Q(6.0 * qv2, 2, 3);
    L(c.l32, 2); L(c.l33, 3); L(c.l34, 4);
  } else if (k == 4) {
    Q(2.0 * v2, 2, 2); Q(4.5 * qv2, 3, 3); Q(3.0 * v2, 1, 3); Q(8.0 * qv, 1, 4); Q(12.0 * qv, 2, 3); Q(8.0 * qv2, 2, 4);
    L(c.l43, 3); L(c.l44, 4);
  }
  return r;
}

// f_k(Y) for this lane's row; Y = the point's stage vector in shared memory.  Branch-free: rows shorter than 6 + 4 terms are padded with
// zero coefficients on an entry the row already reads (make_lane_row), so every lane of the warp runs the same instruction stream.
template <int N>
__device__ __forceinline__ cd lane_rhs(const LaneRow<N>& r, const cd* __restrict__ Y) {
  cd acc = r.q[0] * (Y[r.qi[0]] * Y[r.qj[0]]);
#pragma unroll
  for (int t = 1; t < (N == 5 ? 6 : 3); ++t) acc = acc + r.q[t] * (Y[r.qi[t]] * Y[r.qj[t]]);
#pragma unroll
  for (int t = 0; t < (N == 5 ? 4 : 2); ++t) acc = acc + r.l[t] * Y[r.li[t]];
  return acc + r.h;
}

constexpr int kLaneWarpsPerBlock = 1;

template <int N>
__global__ void __launch_bounds__(32 * kLaneWarpsPerBlock, 1) logsv_mgf_lanes_kernel(
    const cd* __restrict__ phi, const cd* __restrict__ psi, int P, int M, const ChainSpec* __restrict__ spec, const cd* __restrict__ a_in,
    cd* __restrict__ a_out, cd* __restrict__ log_mgf, double y, int* __restrict__ status_out, const double* __restrict__ yb, int phi_stride) {
  constexpr int LPP = N == 5 ? 8 : 4;             // lanes per grid point
  constexpr int PPW = 32 / LPP;                   // points per warp
  constexpr unsigned FULL = 0xffffffffu;
  constexpr double B[6] = {35.0 / 384, 0, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84};
  constexpr double E[7] = {-71.0 / 57600, 0, 71.0 / 16695, -71.0 / 1920, 17253.0 / 339200, -22.0 / 525, 1.0 / 40};
  constexpr double A[6][5] = {{0, 0, 0, 0, 0},
                              {1.0 / 5, 0, 0, 0, 0},
                              {3.0 / 40, 9.0 / 40, 0, 0, 0},
                              {44.0 / 45, -56.0 / 15, 32.0 / 9, 0, 0},
                              {19372.0 / 6561, -25360.0 / 2187, 64448.0 / 6561, -212.0 / 729, 0},
                              {9017.0 / 3168, -355.0 / 33, 46732.0 / 5247, 49.0 / 176, -5103.0 / 18656}};
  __shared__ cd Ysh[kLaneWarpsPerBlock][PPW][N];
  __shared__ double Nsh[kLaneWarpsPerBlock][PPW][N];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int g = lane / LPP, k = lane % LPP;        // point within the warp, component
  const int p = (blockIdx.x * kLaneWarpsPerBlock + wib) * PPW + g;
  {
    const size_t b = blockIdx.y;
    spec += b * M;
    phi += b * (size_t)phi_stride;
    a_out += b * (size_t)M * P * N;
    log_mgf += b * (size_t)M * P;
    if (status_out) status_out += b * (size_t)P;
    if (yb) y = yb[b];
  }
  const bool valid = p < P, comp = k < N, mine = valid && comp;
  const int pc = valid ? p : P - 1;                // out-of-range groups shadow the last point (never stored)
  const int kc = comp ? k : 0;
  cd* Y = &Ysh[wib][g][0];
  double* Nn = &Nsh[wib][g][0];
  const cd ph = phi[pc], ps = psi ? psi[pc] : mk(0.0);
  cd yk = a_in ? a_in[(size_t)pc * N + kc] : mk(0.0);
  const double y2 = y * y;
  const double ys[5] = {1.0, y, y2, y2 * y, y2 * y2};
  int st_all = 0;

  // sum over the point's components, in component order, of this lane's value (identical in every lane of the point)
  auto point_norm = [&](cd v, double inv_scale) -> double {
    const double re = v.re * inv_scale, im = v.im * inv_scale;
    __syncwarp(FULL);
    if (comp) Nn[k] = re * re + im * im;
    __syncwarp(FULL);
    double s = 0.0;
#pragma unroll
    for (int c = 0; c < N; ++c) s += Nn[c];
    return ctrl_sqrt(s) * (N == 5 ? 0.44721359549995793 : 0.57735026918962576);   // / sqrt(N)
  };
  // f_k at the point's vector whose k-th entry is `mine_k`
  auto eval = [&](const LaneRow<N>& row, cd mine_k) -> cd {
    __syncwarp(FULL);
    if (comp) Y[k] = mine_k;
    __syncwarp(FULL);
    return lane_rhs<N>(row, Y);
  };

  for (int mm = 0; mm < M; ++mm) {
    const LogsvModel model = spec[mm].model;
    const double T = spec[mm].dtau;
    const LaneRow<N> row = make_lane_row<N>(kc, model, ph, ps);
    cd K[7];
    K[0] = eval(row, yk);
    double h_abs;
    {   // select_initial_step (scipy/integrate/_ivp/common.py:109-134)
      const double inv_scale = ctrl_rcp(kAtol + cmod(yk) * kRtol);
      const double d0 = point_norm(yk, inv_scale), d1 = point_norm(K[0], inv_scale);
      double h0 = (d0 < 1e-5 || d1 < 1e-5) ? 1e-6 : 0.01 * d0 / d1;
      h0 = fmin(h0, T);
      const cd f1 = eval(row, yk + h0 * K[0]);
      const double d2 = point_norm(f1 - K[0], inv_scale) / h0;
      const double h1 = (d1 <= 1e-15 && d2 <= 1e-15) ? fmax(1e-6, h0 * 1e-3) : exp(0.2 * log(0.01 / fmax(d1, d2)));
      h_abs = fmin(fmin(100.0 * h0, h1), T);
    }
    double t = 0.0, min_step = 0.0;
    bool done = !(t < T), in_step = false, rejected = false;
    int status = 0;
    for (int guard = 0; guard < 1000000 && __any_sync(FULL, !done); ++guard) {
      if (!done && !in_step) {                      // head of the outer loop of rk.py:111-170
        min_step = 10.0 * (__longlong_as_double(__double_as_longlong(t) + 1) - t);
        if (h_abs < min_step) h_abs = min_step;
        rejected = false;
        in_step = true;
      }
      if (!done && h_abs < min_step) {
        status = 1;
        done = true;
      }
      double t_new = t + h_abs;
      if (t_new - T > 0.0) t_new = T;
      const double h = t_new - t;
      if (!done) h_abs = fabs(h);
#pragma unroll
      for (int s = 1; s < 6; ++s) {
        cd acc = K[0] * A[s][0];
#pragma unroll
        for (int jj = 1; jj < 5; ++jj)
          if (jj < s) acc = acc + K[jj] * A[s][jj];
        K[s] = eval(row, yk + acc * h);
      }
      cd acc = K[0] * B[0];
#pragma unroll
      for (int jj = 2; jj < 6; ++jj) acc = acc + K[jj] * B[jj];
      const cd yn = yk + h * acc;
      K[6] = eval(row, yn);
      const double inv_scale = ctrl_rcp(kAtol + fmax(cmod(yk), cmod(yn)) * kRtol);
      cd e = K[0] * E[0];
#pragma unroll
      for (int jj = 2; jj < 6; ++jj) e = e + K[jj] * E[jj];
      const cd err = (e + K[6] * E[6]) * h;
      const double en = point_norm(err, inv_scale);
      if (!done) {
        if (en < 1.0) {
          double factor = en == 0.0 ? 10.0 : fmin(10.0, 0.9 * pow_m02(en));
          if (rejected) factor = fmin(1.0, factor);
          h_abs *= factor;
          t = t_new;
          yk = yn;
          K[0] = K[6];                               // FSAL
          in_step = false;
          done = !(t < T);
        } else {
          h_abs *= fmax(0.2, 0.9 * pow_m02(en));
          rejected = true;
        }
      }
    }
    st_all |= status;
    // outputs of this maturity: a_t1 and log_mgf = sum_k A_k ys_k in component order (affine_expansion.py:674-685)
    __syncwarp(FULL);
    if (comp) Y[k] = yk;
    __syncwarp(FULL);
    if (mine) a_out[((size_t)mm * P + p) * N + k] = yk;
    if (valid && k == 0) {
      cd lm = mk(0.0);
#pragma unroll
      for (int c = 0; c < N; ++c) lm = lm + Y[c] * ys[c];
      log_mgf[(size_t)mm * P + p] = lm;
    }
  }
  if (status_out && valid && k == 0) status_out[p] = st_all;
}

// --------------------------------------------------------------------------------------------------------------------
// Heston closed form: pricers/heston_pricer.py:199-214, chained over maturities with (a, b) carried in registers
// --------------------------------------------------------------------------------------------------------------------
// Written once over the number type: T = cd for the prices, dcd (one direction) for the tangents, hcd (a pair) for the Hessian, with the
// parameters in R = double, dcd, hcd and the overloads sqrt_ / exp_ / log_ of each type.  The constructor is the per-point set-up, step()
// carries (a, b) over one maturity increment; operand order is part of the result (every kernel reproduces the fp64 of the others).
template <class R, class T>
struct HestonClosedForm {
  struct AB {
    T a, b;
  };
  R th, ka, vv2;
  T psi_p, psi_m, zeta, two_zeta;

  __device__ __forceinline__ HestonClosedForm(R theta, R kappa, R rho, R volvol, cd ph, cd ps)
      : th(theta), ka(kappa), vv2(volvol * volvol) {
    const T b1 = T{kappa} + (rho * volvol) * T{ph};
    const T b0 = T{(0.5 * ph) * (ph + mk(1.0)) - ps};
    zeta = sqrt_(b1 * b1 - (2.0 * b0) * vv2);
    psi_p = zeta - b1;
    psi_m = b1 + zeta;
    two_zeta = 2.0 * zeta;
  }
  // Tau: double, or dcd for the theta kernel, which seeds d tau = 1
  template <class Tau>
  __device__ __forceinline__ void step(Tau tau, T& a, T& b) const {
    const T ez = exp_(-(tau * zeta));
    const T c_p = (psi_p + vv2 * b) / two_zeta, c_m = (psi_m - vv2 * b) / two_zeta;
    const T den = c_p * ez + c_m;
    const T b_new = -((-(psi_m * c_p)) * ez + psi_p * c_m) / (vv2 * den);
    const T a_new = (-((th * ka) / vv2)) * (tau * psi_p + 2.0 * log_(den)) + a;
    a = a_new;
    b = b_new;
  }
  // step() on copies of (a, b), returned: what heston_mgf_kernel calls, since stepping its own (a, b) in place gives the same arithmetic on
  // differently allocated registers
  __device__ __forceinline__ AB stepped(double tau, T a, T b) const {
    step(tau, a, b);
    return AB{a, b};
  }
};

__global__ void heston_mgf_kernel(const cd* __restrict__ phi, const cd* __restrict__ psi, int P, int M,
                                  const double* __restrict__ dtaus, b200sv_heston_params hp, const cd* __restrict__ a_in,
                                  const cd* __restrict__ b_in, cd* __restrict__ a_out, cd* __restrict__ b_out,
                                  cd* __restrict__ log_mgf, const b200sv_heston_params* __restrict__ hpb = nullptr, int phi_stride = 0) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  if (hpb) {                                       // batch of parameter sets (b200sv_heston_price_chain_batch): blockIdx.y = set
    const size_t b = blockIdx.y;
    hp = hpb[b];
    phi += b * (size_t)phi_stride;
    log_mgf += b * (size_t)M * P;
  }
  const cd ph = phi[p], ps = psi ? psi[p] : mk(0.0);
  cd a = a_in ? a_in[p] : mk(0.0), b = b_in ? b_in[p] : mk(0.0);
  const HestonClosedForm<double, cd> cf(hp.theta, hp.kappa, hp.rho, hp.volvol, ph, ps);
  for (int mm = 0; mm < M; ++mm) {
    const auto ab = cf.stepped(dtaus[mm], a, b);
    a = ab.a;
    b = ab.b;
    if (a_out) a_out[(size_t)mm * P + p] = a;
    if (b_out) b_out[(size_t)mm * P + p] = b;
    log_mgf[(size_t)mm * P + p] = a + b * hp.v0;
  }
}

// --------------------------------------------------------------------------------------------------------------------
// Fourier sums: utils/mgf_pricer.py:190-219.  One CTA per strike.
// --------------------------------------------------------------------------------------------------------------------
struct StrikeSpec {   // one strike of the chain, with its maturity's forward, discount factor and maturity
  double strike, forward, discfactor;
  int type;     // B200SV_CALL ..
  int slice;    // which log_mgf row
  double ttm;   // only for the fused Black inversion of the batched pricers
  int grid;     // which phi row (batched pricers with per-set grids), else 0
};

constexpr int kFourierThreads = 256;

// The strike sum of one CTA: the quadrature step dp = h3 w_j of every grid point j (the block's threads strided over the P points) goes to
// term(j, dp, phi_j), which adds the point's terms into the zeroed acc[NV] and skips the point itself when its price term is NaN
// (np.nansum); then the fixed-order block_sum leaves the sums in thread 0's acc.
template <int NV, class Term>
__device__ __forceinline__ void strike_sum(const cd* __restrict__ phi, int P, double (&acc)[NV], Term term) {
  __shared__ double red[NV * (kFourierThreads / 32)];
  const double h3 = (phi[1].im - phi[0].im) / 3.0;
  for (int j = threadIdx.x; j < P; j += kFourierThreads) {
    // legacy Simpson weights (utils/mgf_pricer.py:163-170): 1,4,2,4,... with first/last = 1 and THEN every odd index = 4
    const double wq = (j & 1) ? 4.0 : ((j == 0 || j == P - 1) ? 1.0 : 2.0);
    term(j, h3 * wq, phi[j]);
  }
  block_sum<NV, kFourierThreads>(acc, red);
}

__global__ void __launch_bounds__(kFourierThreads) fourier_vanilla_kernel(const cd* __restrict__ log_mgf, const cd* __restrict__ phi,
                                                                         int P, const StrikeSpec* __restrict__ specs,
                                                                         int is_spot, int half_re, double* __restrict__ prices,
                                                                         double* __restrict__ ivols = nullptr) {
  const StrikeSpec sp = specs[blockIdx.x];
  const cd* lm = log_mgf + (size_t)sp.slice * P;
  const double x = log(sp.forward / sp.strike);
  double acc[1] = {};
  strike_sum(phi + (size_t)sp.grid * P, P, acc, [&](int j, double dp, cd ph) {
    cd w;
    if (half_re) {
      w = mk((dp / M_PI) / (ph.im * ph.im + 0.25));
    } else {
      const cd den = is_spot ? (ph + mk(1.0)) * ph : (ph - mk(1.0)) * ph;
      w = -(mk(dp / M_PI) / den);
    }
    const cd term = w * cexp_(lm[j] - x * ph);
    if (term.re == term.re) acc[0] += term.re;
  });
  if (threadIdx.x == 0) {
    const double capped = acc[0], F = sp.forward, K = sp.strike, df = sp.discfactor;
    double price;
    if (is_spot)
      price = sp.type == B200SV_CALL ? df * (F - K * capped) : df * (K - K * capped);
    else
      price = (sp.type == B200SV_CALL || sp.type == B200SV_INV_CALL) ? F * df * (1.0 - capped) : F * df * (exp(-x) - capped);
    prices[blockIdx.x] = price;
    // calibration objective: the Black inversion that follows every chain pricing (option_chain.py:327-346), fused
    if (ivols) ivols[blockIdx.x] = black_implied_vol(F, K, sp.ttm, df, price, sp.type);
  }
}

// Generic Fourier sum  S = nansum_j Re( w_j * exp(coef * g_j + log_mgf_j) )  for the other inversion formulas of
// utils/mgf_pricer.py: options on quadratic variance (:323-358), densities (:361-384), digitals (:224-269).
enum { kModeQvar = 1, kModePdf = 2, kModeDigital = 3 };
struct SumSpec {
  double coef;        // QVAR: strike*ttm ; PDF: z = (x - shift)/scale ; DIGITAL: -ln(F/K)
  double a, b;        // QVAR: a = discfactor, b = ttm ; DIGITAL: a = discfactor
  int type, slice;
};

__global__ void __launch_bounds__(kFourierThreads) fourier_sum_kernel(const cd* __restrict__ log_mgf, const cd* __restrict__ grid, int P,
                                                                     const SumSpec* __restrict__ specs, int mode, int all_calls,
                                                                     double* __restrict__ out) {
  const SumSpec sp = specs[blockIdx.x];
  const cd* lm = log_mgf + (size_t)sp.slice * P;
  double acc[1] = {};
  strike_sum(grid, P, acc, [&](int j, double dp, cd g) {
    cd w;
    if (mode == kModeQvar)
      w = mk(dp / M_PI) / (g * g);                              // (dp/pi)/(psi*psi), :344
    else if (mode == kModePdf)
      w = mk(dp / M_PI);                                        // dp/pi, :374-376
    else
      w = all_calls ? -(mk(dp / M_PI) / g) : (mk(dp / M_PI) / g);   // -/+ (dp/pi)/phi, :241-246
    const cd term = w * cexp_(sp.coef * g + lm[j]);
    if (term.re == term.re) acc[0] += term.re;
  });
  if (threadIdx.x == 0) {
    const double S = acc[0];
    double r;
    if (mode == kModeQvar)
      r = fmax(sp.a * S / sp.b, 1e-10);                         // np.maximum(discfactor*option_price/ttm, 1e-10), :347
    else if (mode == kModePdf)
      r = S;
    else {
      const bool is_call = sp.type == B200SV_CALL;
      r = sp.a * ((is_call == (all_calls != 0)) ? S : 1.0 - S);  // :251-264
    }
    out[blockIdx.x] = r;
  }
}

// --------------------------------------------------------------------------------------------------------------------
// Hawkes jump-diffusion Fourier route (pricers/hawkes_jd_pricer.py:365-641): Riccati system for (a0, a_p, a_m) per transform point,
//   a0' = kappa_p theta_p a_p + kappa_m theta_m a_m + sigma^2 ((phi + 1) phi / 2 - psi)
//   a_p' = E_p(phi - beta1_p a_p - beta1_m a_m) - 1 - kappa_p a_p + comp_p phi        E(z) = exp(-shift z) / (1 + mean z): the jump-size MGF
//   a_m' = E_m(phi - beta2_p a_p - beta2_m a_m) - 1 - kappa_m a_m + comp_m phi        comp = exp(shift) / (1 - mean) - 1
// integrated per maturity by the SAME SciPy-RK45 clone as the LogSV coefficient ODEs (solve_ivp defaults, :636-639), A carried over the
// maturities (:396-416); log-MGF = a0 + a_p lambda_p + a_m lambda_m (:546).  One thread = one transform point.
// --------------------------------------------------------------------------------------------------------------------
struct HawkesMgfConsts {
  double sigma2, shift_p, mean_p, shift_m, mean_m, comp_p, comp_m;
  double kt_p, kt_m, kappa_p, kappa_m, beta1_p, beta1_m, beta2_p, beta2_m, lambda_p, lambda_m;
};

static HawkesMgfConsts make_hawkes_mgf_consts(const b200sv_hawkes_params& p) {
  HawkesMgfConsts c;
  c.sigma2 = p.sigma * p.sigma;
  c.shift_p = p.shift_p;
  c.mean_p = p.mean_p;
  c.shift_m = p.shift_m;
  c.mean_m = p.mean_m;
  c.comp_p = std::exp(p.shift_p) / (1.0 - p.mean_p) - 1.0;
  c.comp_m = std::exp(p.shift_m) / (1.0 - p.mean_m) - 1.0;
  c.kt_p = p.kappa_p * p.theta_p;
  c.kt_m = p.kappa_m * p.theta_m;
  c.kappa_p = p.kappa_p;
  c.kappa_m = p.kappa_m;
  c.beta1_p = p.beta1_p;
  c.beta1_m = p.beta1_m;
  c.beta2_p = p.beta2_p;
  c.beta2_m = p.beta2_m;
  c.lambda_p = p.lambda_p;
  c.lambda_m = p.lambda_m;
  return c;
}

struct HawkesRhsFn {
  const HawkesMgfConsts& c;
  cd phi, drift0;          // drift0 = sigma^2 ((phi + 1) phi / 2 - psi)
  __device__ __forceinline__ void operator()(const cd (&A)[3], cd (&out)[3]) const {
    const cd zp = (phi - c.beta1_p * A[1]) - c.beta1_m * A[2], zm = (phi - c.beta2_p * A[1]) - c.beta2_m * A[2];
    const cd jp = exp_(-c.shift_p * zp) / (mk(1.0) + c.mean_p * zp) - mk(1.0);
    const cd jm = exp_(-c.shift_m * zm) / (mk(1.0) + c.mean_m * zm) - mk(1.0);
    out[0] = (c.kt_p * A[1] + c.kt_m * A[2]) + drift0;
    out[1] = (jp - c.kappa_p * A[1]) + c.comp_p * phi;
    out[2] = (jm - c.kappa_m * A[2]) + c.comp_m * phi;
  }
};

// a_io: A(0) per point or nullptr (zeros); restart != 0: every maturity starts from A = 0 and integrates over ITS ttm (the risk-kernel
// normalisers, :498-509) instead of carrying A over the increments
template <int TPB>
__global__ void __launch_bounds__(TPB) hawkes_mgf_kernel(const cd* __restrict__ phi, const cd* __restrict__ psi, int P, int M,
                                                         const double* __restrict__ dtaus, HawkesMgfConsts c, const cd* __restrict__ a_in,
                                                         cd* __restrict__ a_out, cd* __restrict__ log_mgf, int restart, int* __restrict__ status) {
  __shared__ cd stage_smem[6 * 3 * TPB];
  const int p = blockIdx.x * TPB + threadIdx.x;
  if (p >= P) return;
  StageStore<3, TPB> K{stage_smem + threadIdx.x};
#pragma unroll
  for (int i = 0; i < 18; ++i) stage_smem[threadIdx.x + i * TPB] = mk(0.0);
  cd A[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) A[k] = a_in ? a_in[(size_t)p * 3 + k] : mk(0.0);
  const cd ph = phi[p], ps = psi ? psi[p] : mk(0.0);
  const HawkesRhsFn f{c, ph, c.sigma2 * (0.5 * ((ph + mk(1.0)) * ph) - ps)};
  int st = 0;
  for (int m = 0; m < M; ++m) {
    if (restart) {
#pragma unroll
      for (int k = 0; k < 3; ++k) A[k] = mk(0.0);
    }
    st |= rk45_generic<3, TPB>(A, dtaus[m], f, K, nullptr);
    if (a_out) {
#pragma unroll
      for (int k = 0; k < 3; ++k) a_out[((size_t)m * P + p) * 3 + k] = A[k];
    }
    log_mgf[(size_t)m * P + p] = (A[0] + A[1] * c.lambda_p) + A[2] * c.lambda_m;
  }
  if (status) status[p] = st;
}

// ---- several Hawkes parameter sets in one Riccati launch (b200sv_hawkesjd_price_chains_batch, DESIGN.md §4.10) ----
// hawkes_mgf_kernel reads its constants as kernel parameters, and ptxas contracts HawkesRhsFn's plain fp64 products and sums around
// them: it sinks the loop-invariant sigma^2 drift and comp * phi products into fused multiply-adds inside the step loop, fuses the
// A-products of z and of the outputs, and leaves Smith's division unfused.  With the constants in registers it hoists those products
// instead, and rows move by an ulp.  So the set-major kernel's right-hand side spells out, with rounding intrinsics that ptxas may
// neither fuse nor split, the operations hawkes_mgf_kernel's SASS performs, and the two kernels carry the same fp64 instructions
// (DESIGN.md §4.10).  exp_ (sincos, exp) is shared.

// Smith's division as operator/ compiles in HawkesRhsFn: every product and sum rounded on its own
__device__ __forceinline__ cd cdiv_rn(cd a, cd b) {
  if (fabs(b.re) >= fabs(b.im)) {
    const double r = __ddiv_rn(b.im, b.re), d = __dadd_rn(b.re, __dmul_rn(b.im, r));
    return cd{__ddiv_rn(__dadd_rn(a.re, __dmul_rn(a.im, r)), d), __ddiv_rn(__dsub_rn(a.im, __dmul_rn(a.re, r)), d)};
  }
  const double r = __ddiv_rn(b.re, b.im), d = __dadd_rn(__dmul_rn(b.re, r), b.im);
  return cd{__ddiv_rn(__dadd_rn(__dmul_rn(a.re, r), a.im), d), __ddiv_rn(__dsub_rn(__dmul_rn(a.im, r), a.re), d)};
}

// E(z) - 1 of HawkesRhsFn: exp(-shift z) / (1 + mean z) - 1
__device__ __forceinline__ cd hawkes_jump_rn(cd z, double shift, double mean) {
  const cd q = cdiv_rn(exp_(cd{__dmul_rn(-shift, z.re), __dmul_rn(-shift, z.im)}), cd{__fma_rn(z.re, mean, 1.0), __fma_rn(z.im, mean, 0.0)});
  return cd{__dadd_rn(q.re, -1.0), q.im};
}

// HawkesRhsFn for constants in registers.  d = (phi + 1) phi / 2 - psi with psi = 0: the sigma^2 product of drift0 is fused into out[0].
struct HawkesSetsRhsFn {
  const HawkesMgfConsts& c;
  cd phi, d;
  __device__ __forceinline__ void operator()(const cd (&A)[3], cd (&out)[3]) const {
    const cd zp{__fma_rn(-c.beta1_m, A[2].re, __fma_rn(-c.beta1_p, A[1].re, phi.re)),
                __fma_rn(-c.beta1_m, A[2].im, __fma_rn(-c.beta1_p, A[1].im, phi.im))};
    const cd zm{__fma_rn(-c.beta2_m, A[2].re, __fma_rn(-c.beta2_p, A[1].re, phi.re)),
                __fma_rn(-c.beta2_m, A[2].im, __fma_rn(-c.beta2_p, A[1].im, phi.im))};
    const cd jp = hawkes_jump_rn(zp, c.shift_p, c.mean_p), jm = hawkes_jump_rn(zm, c.shift_m, c.mean_m);
    out[0] = cd{__fma_rn(d.re, c.sigma2, __fma_rn(A[1].re, c.kt_p, __dmul_rn(A[2].re, c.kt_m))),
                __fma_rn(d.im, c.sigma2, __fma_rn(A[1].im, c.kt_p, __dmul_rn(A[2].im, c.kt_m)))};
    out[1] = cd{__fma_rn(phi.re, c.comp_p, __fma_rn(-A[1].re, c.kappa_p, jp.re)), __fma_rn(phi.im, c.comp_p, __fma_rn(-A[1].im, c.kappa_p, jp.im))};
    out[2] = cd{__fma_rn(phi.re, c.comp_m, __fma_rn(-A[2].re, c.kappa_m, jm.re)), __fma_rn(phi.im, c.comp_m, __fma_rn(-A[2].im, c.kappa_m, jm.im))};
  }
};

// One thread = one (set, transform point) of B sets sharing the maturity increments dtaus [M]: the set is the FASTEST thread index (the
// logsv_mgf_kernel batch mapping: the lanes of a warp integrate one point for neighbouring sets, which take nearly the same steps).
// consts [B], phi [B][P] (phi_stride = P) or one grid (0); log_mgf [B][M][P].  A starts at 0 and is carried over the maturities.
// Every value equals hawkes_mgf_kernel's for that set alone, bit for bit, whatever block size either runs at.
// RESTART: hawkes_mgf_kernel's restart mode for sets of different maturity counts (the risk-kernel normalisers of several chains, DESIGN.md
// §4.11).  Set b owns the rows set_m0[b] .. set_m0[b + 1] - 1: every row restarts from A = 0 and integrates over its full maturity
// dtaus[row] (the set's chain's ttms, one copy per set), and log_mgf is [rows][P]; M is not read.
template <int TPB, bool RESTART = false>
__global__ void __launch_bounds__(TPB) hawkes_mgf_sets_kernel(const cd* __restrict__ phi, int P, int M, const double* __restrict__ dtaus,
                                                              const HawkesMgfConsts* __restrict__ consts, int B, int phi_stride,
                                                              cd* __restrict__ log_mgf, const int* __restrict__ set_m0 = nullptr) {
  __shared__ cd stage_smem[6 * 3 * TPB];
  const long long t = (long long)blockIdx.x * TPB + threadIdx.x;
  if (t >= (long long)B * P) return;
  const int b = (int)(t % B), p = (int)(t / B);
  const HawkesMgfConsts c = consts[b];
  StageStore<3, TPB> K{stage_smem + threadIdx.x};
#pragma unroll
  for (int i = 0; i < 18; ++i) stage_smem[threadIdx.x + i * TPB] = mk(0.0);
  cd A[3] = {mk(0.0), mk(0.0), mk(0.0)};
  const cd ph = phi[(size_t)b * phi_stride + p];
  const cd p1{__dadd_rn(ph.re, 1.0), __dadd_rn(ph.im, 0.0)};                                    // phi + 1
  const cd pp{__fma_rn(p1.re, ph.re, -__dmul_rn(p1.im, ph.im)), __fma_rn(p1.re, ph.im, __dmul_rn(p1.im, ph.re))};   // (phi + 1) phi
  const HawkesSetsRhsFn f{c, ph, cd{__fma_rn(pp.re, 0.5, -0.0), __fma_rn(pp.im, 0.5, -0.0)}};
  if (RESTART) {
    const int m0 = set_m0[b];
    M = set_m0[b + 1] - m0;
    dtaus += m0;
    log_mgf += (size_t)m0 * P;
  } else {
    log_mgf += (size_t)b * M * P;
  }
  cd* lm = log_mgf + p;
  for (int m = 0; m < M; ++m) {
    if (RESTART) {
#pragma unroll
      for (int k = 0; k < 3; ++k) A[k] = mk(0.0);
    }
    rk45_generic<3, TPB>(A, dtaus[m], f, K, nullptr);
    lm[(size_t)m * P] = cd{__fma_rn(A[2].re, c.lambda_m, __fma_rn(A[1].re, c.lambda_p, A[0].re)),
                           __fma_rn(A[2].im, c.lambda_m, __fma_rn(A[1].im, c.lambda_p, A[0].im))};
  }
}

// slice_pricer_with_mgf_grid_with_gamma (utils/mgf_pricer.py:273-320): general weights -(dp/pi) / ((phi + g + 1)(phi + g)) (its fast branch
// compares Re(phi) with +(1/2 + g) while the grid sits on -(1/2 + g), so it never runs), calls gamma_forward - n K^(1+g) S, puts K - n K^(1+g) S;
// no discount factor (both as in the reference).  Row grid sp.grid sits on Re phi = -1/2 - gammas[sp.grid]; norm_gfwd[2 sp.slice + {0, 1}] =
// that slice's normaliser n and forward under the risk kernel (b200sv_fourier_gamma: one grid and one slice).  ivols (optional): the Black
// inversion of fourier_vanilla_kernel fused for the batch -- spec.forward / discfactor / ttm are the chain's own, and the calibration
// objective inverts the (undiscounted) gamma price with them (compute_model_ivols_from_chain_data, as in the reference).
__global__ void __launch_bounds__(kFourierThreads) fourier_gamma_batch_kernel(const cd* __restrict__ log_mgf, const cd* __restrict__ phi, int P,
                                                                             const StrikeSpec* __restrict__ specs, const double* __restrict__ gammas,
                                                                             const double* __restrict__ norm_gfwd, double* __restrict__ prices,
                                                                             double* __restrict__ ivols) {
  __shared__ double red[kFourierThreads / 32];
  const StrikeSpec sp = specs[blockIdx.x];
  const double gamma = gammas[sp.grid];
  const cd* lm = log_mgf + (size_t)sp.slice * P;
  phi += (size_t)sp.grid * P;
  const double x = log(sp.forward / sp.strike);
  const double h3 = (phi[1].im - phi[0].im) / 3.0;
  const bool fast = fabs(phi[0].re - (0.5 + gamma)) < 1e-10;
  double acc[1] = {0.0};
  for (int j = threadIdx.x; j < P; j += kFourierThreads) {
    const double wq = (j & 1) ? 4.0 : ((j == 0 || j == P - 1) ? 1.0 : 2.0);
    const double dp = h3 * wq;
    const cd ph = phi[j];
    const cd pg = ph + mk(gamma);
    const cd w = fast ? mk((dp / M_PI) / (ph.im * ph.im + 0.25)) : -(mk(dp / M_PI) / ((pg + mk(1.0)) * pg));
    const cd term = w * cexp_(lm[j] - x * ph);
    if (term.re == term.re) acc[0] += term.re;
  }
  block_sum<1, kFourierThreads>(acc, red);
  if (threadIdx.x == 0) {
    const double gk = pow(sp.strike, 1.0 + gamma), normalizer = norm_gfwd[2 * (size_t)sp.slice], gamma_forward = norm_gfwd[2 * (size_t)sp.slice + 1];
    const double price = (sp.type == B200SV_CALL ? gamma_forward : sp.strike) - normalizer * gk * acc[0];
    prices[blockIdx.x] = price;
    if (ivols) ivols[blockIdx.x] = black_implied_vol(sp.forward, sp.strike, sp.ttm, sp.discfactor, price, sp.type);
  }
}

// --------------------------------------------------------------------------------------------------------------------
// Forward-mode sensitivities of the Fourier chain pricers (DESIGN.md §4.2)
// --------------------------------------------------------------------------------------------------------------------
// d(LogsvModel field) / d(one parameter), built on the host (make_model_tangents); eta2 does not depend on the parameters.
struct LogsvModelTangent {
  double theta, th2, v2, qv, qv2, lam, k2p, kp, beta_eta;
};
constexpr int kLogsvOdeDirs = 5;     // theta, kappa1, kappa2, beta, volvol (sigma0 enters only through y = sigma0 - theta)
constexpr int kHestonOdeDirs = 4;    // theta, kappa, rho, volvol (v0 enters only through log_mgf = a + b v0)

// make_model differentiated field by field; kappa2 is held fixed when kappa1 or theta moves
static void make_model_tangents(const b200sv_logsv_params& p, double eta, bool spot, LogsvModelTangent (&d)[kLogsvOdeDirs]) {
  for (auto& t : d) t = LogsvModelTangent{0, 0, 0, 0, 0, 0, 0, 0, 0};
  const double v2 = p.beta * p.beta + p.volvol * p.volvol, th2 = p.theta * p.theta;
  LogsvModelTangent& th = d[0];      // theta
  th.theta = 1.0;
  th.th2 = 2.0 * p.theta;
  th.qv = v2;
  th.qv2 = 2.0 * p.theta * v2;
  th.lam = spot ? 0.0 : 2.0 * p.beta * p.theta * eta;
  th.kp = spot ? p.kappa2 : p.kappa2 - 2.0 * p.beta * eta;
  d[1].kp = 1.0;                     // kappa1
  d[2].k2p = 1.0;                    // kappa2
  d[2].kp = p.theta;
  LogsvModelTangent& be = d[3];      // beta
  be.v2 = 2.0 * p.beta;
  be.qv = 2.0 * p.beta * p.theta;
  be.qv2 = 2.0 * p.beta * th2;
  be.lam = spot ? 0.0 : th2 * eta;
  be.k2p = spot ? 0.0 : -eta;
  be.kp = spot ? 0.0 : -2.0 * p.theta * eta;
  be.beta_eta = eta;
  LogsvModelTangent& vv = d[4];      // volvol
  vv.v2 = 2.0 * p.volvol;
  vv.qv = 2.0 * p.volvol * p.theta;
  vv.qv2 = 2.0 * p.volvol * th2;
}

// make_coef differentiated: linear in the model fields except the products th2 * beta_eta, theta * beta_eta (in b) and th2 * eta2,
// theta * eta2 (in h0, h1), which take the product rule
__device__ __forceinline__ Coef make_dcoef(const LogsvModel& m, const LogsvModelTangent& d, cd phi, cd psi) {
  Coef c;
  const cd b = m.beta_eta * phi, db = d.beta_eta * phi;
  const cd dtb = d.th2 * b + m.th2 * db;          // d(th2 b)
  const cd d1b = d.theta * b + m.theta * db;      // d(theta b)
  c.l01 = mk(d.lam) - dtb;
  c.l11 = mk(-d.kp) - 2.0 * d1b;
  c.l12 = 2.0 * (mk(d.lam + d.qv) - dtb);
  c.l21 = mk(-d.k2p) - db;
  c.l22 = mk(d.v2 - 2.0 * d.kp) - 4.0 * d1b;
  c.l23 = 3.0 * (mk(2.0 * d.qv) - dtb);
  c.l32 = -2.0 * (mk(d.k2p) + db);
  c.l33 = 3.0 * (mk(d.v2 - d.kp) - 2.0 * d1b);
  c.l34 = 4.0 * (mk(3.0 * d.qv) - dtb);
  c.l43 = -3.0 * (mk(d.k2p) + db);
  c.l44 = 2.0 * (mk(d.v2 - 2.0 * d.kp) - 4.0 * d1b);
  const cd r = m.spot ? phi * (phi + mk(1.0)) - 2.0 * psi : phi * (phi - mk(1.0)) - 2.0 * psi;
  c.h0 = (0.5 * d.th2 * m.eta2) * r;
  c.h1 = (d.theta * m.eta2) * r;
  c.h2 = mk(0.0);
  return c;
}

// The rows of rhs<>() with the products A_i A_j given as q = {11, 12, 22, 13, 14, 23, 24, 33} and the linear inputs as u, H added if
// WithH.  The right-hand side is linear in q, in u and in (v2, qv, qv2, Coef) separately, so both halves of its tangent are this function.
template <int N, int TPB, bool WithH>
__device__ __forceinline__ void rhs_rows(const cd (&q)[8], const cd (&u)[N], double v2, double qv, double qv2, const CoefView<TPB>& cv,
                                         cd (&out)[N]) {
  const cd h0 = WithH ? cv.at(11) : mk(0.0), h1 = WithH ? cv.at(12) : mk(0.0), h2 = WithH ? cv.at(13) : mk(0.0);
  out[0] = (0.5 * qv2) * q[0] + cv.at(0) * u[1] + qv2 * u[2] + h0;
  if constexpr (N == 5) {
    out[1] = qv * q[0] + (2.0 * qv2) * q[1] + cv.at(1) * u[1] + cv.at(2) * u[2] + (3.0 * qv2) * u[3] + h1;
    out[2] = (0.5 * v2) * q[0] + (2.0 * qv2) * q[2] + (4.0 * qv) * q[1] + (3.0 * qv2) * q[3] + cv.at(3) * u[1] + cv.at(4) * u[2] +
             cv.at(5) * u[3] + (6.0 * qv2) * u[4] + h2;
    out[3] = (4.0 * qv) * q[2] + (2.0 * v2) * q[1] + (6.0 * qv) * q[3] + (4.0 * qv2) * q[4] + (6.0 * qv2) * q[5] + cv.at(6) * u[2] +
             cv.at(7) * u[3] + cv.at(8) * u[4];
    out[4] = (2.0 * v2) * q[2] + (4.5 * qv2) * q[7] + (3.0 * v2) * q[3] + (8.0 * qv) * q[4] + (12.0 * qv) * q[5] + (8.0 * qv2) * q[6] +
             cv.at(9) * u[3] + cv.at(10) * u[4];
  } else {
    out[1] = qv * q[0] + (2.0 * qv2) * q[1] + cv.at(1) * u[1] + cv.at(2) * u[2] + h1;
    out[2] = (0.5 * v2) * q[0] + (2.0 * qv2) * q[2] + (4.0 * qv) * q[1] + cv.at(3) * u[1] + cv.at(4) * u[2] + h2;
  }
}

// d f(A) = J(A) dA + d_p f(A):  J(A) dA = rows(products A_i dA_j + dA_i A_j, dA; model, Coef without H) and d_p f(A) = rows(A_i A_j, A;
// d model, d Coef with d H).
template <int N, int TPB>
__device__ __forceinline__ void rhs_tangent(const cd (&A)[N], const cd (&dA)[N], const LogsvModel& m, const CoefView<TPB>& c,
                                            const LogsvModelTangent& dm, const CoefView<TPB>& dc, cd (&out)[N]) {
  const cd z = mk(0.0);
  cd q[8] = {A[1] * A[1], A[1] * A[2], A[2] * A[2], z, z, z, z, z};
  cd dq[8] = {2.0 * (A[1] * dA[1]), A[1] * dA[2] + dA[1] * A[2], 2.0 * (A[2] * dA[2]), z, z, z, z, z};
  if constexpr (N == 5) {
    q[3] = A[1] * A[3]; q[4] = A[1] * A[4]; q[5] = A[2] * A[3]; q[6] = A[2] * A[4]; q[7] = A[3] * A[3];
    dq[3] = A[1] * dA[3] + dA[1] * A[3];
    dq[4] = A[1] * dA[4] + dA[1] * A[4];
    dq[5] = A[2] * dA[3] + dA[2] * A[3];
    dq[6] = A[2] * dA[4] + dA[2] * A[4];
    dq[7] = 2.0 * (A[3] * dA[3]);
  }
  cd jv[N], pv[N];
  rhs_rows<N, TPB, false>(dq, dA, m.v2, m.qv, m.qv2, c, jv);
  rhs_rows<N, TPB, true>(q, A, dm.v2, dm.qv, dm.qv2, dc, pv);
#pragma unroll
  for (int k = 0; k < N; ++k) out[k] = jv[k] + pv[k];
}

// One tangent stepped on rk45_generic's attempts: dY_s = dy + h sum_j a_sj dK_j, dK_s = d f(Y_s), accepted steps commit
// dy <- dy + h sum_j b_j dK_j and dK_0 <- dK_6 (FSAL).  dK: 8 "stages" in shared memory (StageStore indexes (stage * N + k) * TPB, so 8
// stages fit in 8 * N * TPB entries), 0..6 the stage tangents, 7 the candidate dy of the current attempt.  dy stays in registers and
// carries over maturities like A.
template <int N, int TPB>
struct TangentStore {
  StageStore<N, TPB> dK;
  cd dy[N];

  // the input dy + h sum_j a_sj dK_j of stage s
  __device__ __forceinline__ void stage_input(int s, double h, cd (&out)[N]) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      cd acc = dK.at(0, k) * c_A[s][0];
#pragma unroll
      for (int jj = 1; jj < 5; ++jj) acc = acc + dK.at(jj, k) * c_A[s][jj];
      out[k] = dy[k] + acc * h;
    }
  }
  // the candidate dy + h sum_j b_j dK_j of the attempt, also parked in stage 7
  __device__ __forceinline__ void candidate(double h, cd (&out)[N]) {
    constexpr double B[6] = {35.0 / 384, 0, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84};
#pragma unroll
    for (int k = 0; k < N; ++k) {
      cd acc = dK.at(0, k) * B[0];
#pragma unroll
      for (int jj = 2; jj < 6; ++jj) acc = acc + dK.at(jj, k) * B[jj];
      out[k] = dy[k] + h * acc;
      dK.at(7, k) = out[k];
    }
  }
};

// The accept step of the tangent stores of one attempt: dy <- the candidate, dK_0 <- dK_6 (FSAL), component by component across the stores.
template <int N, int TPB, class... Store>
__device__ __forceinline__ void accept_tangents(Store&... s) {
#pragma unroll
  for (int k = 0; k < N; ++k) {
    ((s.dy[k] = s.dK.at(7, k)), ...);
    ((s.dK.at(0, k) = s.dK.at(6, k)), ...);
  }
}

// The tangent of one parameter direction.  TanRhs: functor ``void operator()(const cd (&Y)[N], const cd (&dY)[N], cd (&out)[N]) const``
// = J(Y) dY + d_p f(Y) of one direction (LogsvTanRhsFn, HawkesTanRhsFn); the bookkeeping does not depend on it.
template <int N, int TPB, typename TanRhs>
struct TangentHook {
  TanRhs f;
  TangentStore<N, TPB> t;

  __device__ __forceinline__ void eval(int s, const cd (&Y)[N], const cd (&dY)[N]) {
    cd o[N];
    f(Y, dY, o);
#pragma unroll
    for (int k = 0; k < N; ++k) t.dK.at(s, k) = o[k];
  }
  __device__ __forceinline__ void start(const cd (&y)[N]) { eval(0, y, t.dy); }
  __device__ __forceinline__ void stage(int s, const cd (&yt)[N], double h) {
    cd dyt[N];
    t.stage_input(s, h, dyt);
    eval(s, yt, dyt);
  }
  __device__ __forceinline__ void last(const cd (&yn)[N], double h) {
    cd dyn[N];
    t.candidate(h, dyn);
    eval(6, yn, dyn);
  }
  __device__ __forceinline__ void accept() { accept_tangents<N, TPB>(t); }
};

template <int N, int TPB>
struct LogsvTanRhsFn {
  const LogsvModel* m;
  const CoefView<TPB>* c;
  LogsvModelTangent dm;
  CoefView<TPB> dc;
  __device__ __forceinline__ void operator()(const cd (&Y)[N], const cd (&dY)[N], cd (&out)[N]) const {
    rhs_tangent<N, TPB>(Y, dY, *m, *c, dm, dc, out);
  }
};
template <int N, int TPB>
using LogsvTangentHook = TangentHook<N, TPB, LogsvTanRhsFn<N, TPB>>;

constexpr int kTangentTPB = 16;      // shared memory per thread: 6N primal stages + 8N tangent stages + 2 x 14 coefficients

// One thread = one (grid point, parameter direction): the primal integration of logsv_mgf_kernel (same rk45_generic, same mesh) plus one
// tangent.  The D = 5 directions of a point are neighbouring threads, so a warp runs few meshes.  dspec [M][5]: d(model)/d(direction).
// Outputs: dlog_mgf [6][M][P] (row 0 sigma0, rows 1.. the directions, LOGSV_GREEK_PARAMS order), log_mgf [M][P], status [P], nfev [P].
template <int N>
__global__ void __launch_bounds__(kTangentTPB) logsv_mgf_tangent_kernel(const cd* __restrict__ phi, int P, int M, const ChainSpec* __restrict__ spec,
                                                                         const LogsvModelTangent* __restrict__ dspec, double y,
                                                                         cd* __restrict__ dlog_mgf, cd* __restrict__ log_mgf,
                                                                         int* __restrict__ status, int* __restrict__ nfev) {
  constexpr int TPB = kTangentTPB, D = kLogsvOdeDirs;
  __shared__ cd stage_smem[6 * N * TPB];
  __shared__ cd tan_smem[8 * N * TPB];
  __shared__ cd coef_smem[14 * TPB];
  __shared__ cd dcoef_smem[14 * TPB];
  const int t = blockIdx.x * TPB + threadIdx.x;
  if (t >= P * D) return;
  const int p = t / D, dir = t % D;
#pragma unroll
  for (int i = 0; i < 6 * N; ++i) stage_smem[threadIdx.x + i * TPB] = mk(0.0);
#pragma unroll
  for (int i = 0; i < 8 * N; ++i) tan_smem[threadIdx.x + i * TPB] = mk(0.0);
  StageStore<N, TPB> K{stage_smem + threadIdx.x};
  const CoefView<TPB> c{coef_smem + threadIdx.x};
  LogsvTangentHook<N, TPB> tan;
  tan.f.c = &c;
  tan.f.dc = CoefView<TPB>{dcoef_smem + threadIdx.x};
  tan.t.dK = StageStore<N, TPB>{tan_smem + threadIdx.x};
  cd A[N];
#pragma unroll
  for (int k = 0; k < N; ++k) {
    A[k] = mk(0.0);
    tan.t.dy[k] = mk(0.0);
  }
  const cd ph = phi[p], ps = mk(0.0);
  const double y2 = y * y;
  const double ys[5] = {1.0, y, y2, y2 * y, y2 * y2};
  const double dys[5] = {0.0, 1.0, 2.0 * y, 3.0 * y2, 4.0 * (y2 * y)};      // d ys / d y; dy/dsigma0 = 1, dy/dtheta = -1
  const double dy_dp = dir == 0 ? -1.0 : 0.0;
  int st = 0, nf = 0;
  for (int mm = 0; mm < M; ++mm) {
    const LogsvModel model = spec[mm].model;
    store_coef<TPB>(coef_smem + threadIdx.x, make_coef(model, ph, ps));
    tan.f.m = &model;
    tan.f.dm = dspec[mm * D + dir];
    store_coef<TPB>(dcoef_smem + threadIdx.x, make_dcoef(model, tan.f.dm, ph, ps));
    int nfe = 0;
    st |= rk45_generic<N, TPB>(A, spec[mm].dtau, LogsvRhsFn<N, TPB>{model, c}, K, &nfe, &tan);
    nf += nfe;
    cd lm = mk(0.0), dlm = mk(0.0), dls = mk(0.0);
#pragma unroll
    for (int k = 0; k < N; ++k) {
      lm = lm + A[k] * ys[k];
      dlm = dlm + (tan.t.dy[k] * ys[k] + A[k] * (dys[k] * dy_dp));
      dls = dls + A[k] * dys[k];
    }
    dlog_mgf[((size_t)(1 + dir) * M + mm) * P + p] = dlm;
    if (dir == 0) {
      dlog_mgf[(size_t)mm * P + p] = dls;
      log_mgf[(size_t)mm * P + p] = lm;
    }
  }
  if (dir == 0) {
    if (status) status[p] = st;
    if (nfev) nfev[p] = nf;
  }
}

// dual complex numbers (value, derivative in one direction) for the Heston closed form
struct dcd {
  cd v, d;
};
__device__ __forceinline__ dcd dmk(cd v, cd d = mk(0.0)) { return dcd{v, d}; }
__device__ __forceinline__ dcd operator+(dcd a, dcd b) { return dcd{a.v + b.v, a.d + b.d}; }
__device__ __forceinline__ dcd operator-(dcd a, dcd b) { return dcd{a.v - b.v, a.d - b.d}; }
__device__ __forceinline__ dcd operator-(dcd a) { return dcd{-a.v, -a.d}; }
__device__ __forceinline__ dcd operator*(dcd a, dcd b) { return dcd{a.v * b.v, a.d * b.v + a.v * b.d}; }
__device__ __forceinline__ dcd operator*(double s, dcd a) { return dcd{s * a.v, s * a.d}; }
__device__ __forceinline__ dcd operator/(dcd a, dcd b) {
  const cd q = a.v / b.v;
  return dcd{q, (a.d - q * b.d) / b.v};
}
__device__ __forceinline__ dcd sqrt_(dcd z) {
  const cd s = sqrt_(z.v);
  return dcd{s, z.d / (2.0 * s)};
}
__device__ __forceinline__ dcd exp_(dcd z) {
  const cd e = exp_(z.v);
  return dcd{e, e * z.d};
}
__device__ __forceinline__ dcd log_(dcd z) { return dcd{log_(z.v), z.d / z.v}; }

// heston_mgf_kernel in forward mode: one thread = one (grid point, direction theta | kappa | rho | volvol), (a, b) and their tangents
// carried over the maturities.  dlog_mgf [5][M][P]: row 0 d/dv0 = b, rows 1.. the directions (HESTON_GREEK_PARAMS order).
__global__ void heston_mgf_tangent_kernel(const cd* __restrict__ phi, int P, int M, const double* __restrict__ dtaus, b200sv_heston_params hp,
                                          cd* __restrict__ dlog_mgf) {
  constexpr int D = kHestonOdeDirs;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= P * D) return;
  const int p = t / D, dir = t % D;
  const dcd th = dmk(mk(hp.theta), mk(dir == 0 ? 1.0 : 0.0)), ka = dmk(mk(hp.kappa), mk(dir == 1 ? 1.0 : 0.0));
  const dcd rho = dmk(mk(hp.rho), mk(dir == 2 ? 1.0 : 0.0)), vv = dmk(mk(hp.volvol), mk(dir == 3 ? 1.0 : 0.0));
  const HestonClosedForm<dcd, dcd> cf(th, ka, rho, vv, phi[p], mk(0.0));
  dcd a = dmk(mk(0.0)), b = dmk(mk(0.0));
  for (int mm = 0; mm < M; ++mm) {
    cf.step(dtaus[mm], a, b);
    dlog_mgf[((size_t)(1 + dir) * M + mm) * P + p] = a.d + b.d * hp.v0;
    if (dir == 0) dlog_mgf[(size_t)mm * P + p] = b.v;
  }
}

// ---- Hawkes jump-diffusion (DESIGN.md §4.3) ----
// 15 parameters (HAWKES_GREEK_PARAMS: the HawkesJDParams fields without mu, which the Fourier route never reads, and risk_premia_gamma);
// lambda_p / lambda_m enter only through log_mgf = a0 + a_p lambda_p + a_m lambda_m, the other 13 are ODE directions.
constexpr int kHawkesGreekParams = 15;
constexpr int kHawkesOdeDirs = 13;
// row of dlog_mgf / greeks of ODE direction d (the two lambda rows, 5 and 10, are a_p and a_m)
__host__ __device__ constexpr int hawkes_dir_row(int d) { return d < 5 ? d : d < 9 ? d + 1 : d + 2; }

// d(HawkesMgfConsts field) / d(each ODE direction), built on the host: each direction is a HawkesMgfConsts of field derivatives.
// comp = e^shift / (1 - mean) - 1 is derived: d comp / d shift = e^shift / (1 - mean), d comp / d mean = e^shift / (1 - mean)^2.
struct HawkesTangentDirs {
  HawkesMgfConsts d[kHawkesOdeDirs];
};

static HawkesTangentDirs make_hawkes_tangents(const b200sv_hawkes_params& p) {
  HawkesTangentDirs t;
  for (auto& d : t.d) d = HawkesMgfConsts{0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  const double ep = std::exp(p.shift_p) / (1.0 - p.mean_p), em = std::exp(p.shift_m) / (1.0 - p.mean_m);
  t.d[0].sigma2 = 2.0 * p.sigma;                                     // sigma
  t.d[1].shift_p = 1.0, t.d[1].comp_p = ep;                          // shift_p
  t.d[2].mean_p = 1.0, t.d[2].comp_p = ep / (1.0 - p.mean_p);        // mean_p
  t.d[3].shift_m = 1.0, t.d[3].comp_m = em;                          // shift_m
  t.d[4].mean_m = 1.0, t.d[4].comp_m = em / (1.0 - p.mean_m);        // mean_m
  t.d[5].kt_p = p.kappa_p;                                           // theta_p
  t.d[6].kappa_p = 1.0, t.d[6].kt_p = p.theta_p;                     // kappa_p
  t.d[7].beta1_p = 1.0;                                              // beta1_p
  t.d[8].beta2_p = 1.0;                                              // beta2_p
  t.d[9].kt_m = p.kappa_m;                                           // theta_m
  t.d[10].kappa_m = 1.0, t.d[10].kt_m = p.theta_m;                   // kappa_m
  t.d[11].beta1_m = 1.0;                                             // beta1_m
  t.d[12].beta2_m = 1.0;                                             // beta2_m
  return t;
}

// d E(z) of the jump-size MGF E(z) = e^{-s z} / (1 + m z) along (dz, ds, dm):  E (-(s + m / (1 + m z)) dz - z ds - z / (1 + m z) dm)
__device__ __forceinline__ cd hawkes_djump(cd z, cd dz, double s, double m, double ds, double dm) {
  const cd r = mk(1.0) / (mk(1.0) + m * z);
  const cd e = exp_(-s * z) * r;
  return e * (-((mk(s) + m * r) * dz) - z * (mk(ds) + dm * r));
}

// d f(A) = J(A) dA + d_p f(A) of HawkesRhsFn for one direction, d = d(consts)/d(direction).  Phi adds a move dphi of the transform
// variable (the risk kernel, DESIGN.md §4.12; psi = 0 there, so drift0 = sigma^2 (phi + 1) phi / 2):
// d rhs0 += sigma^2 (phi + 1/2) dphi,  dz_p = dz_m += dphi,  d rhs1 += comp_p dphi,  d rhs2 += comp_m dphi.
template <bool Phi>
struct HawkesTanRhsFn {
  const HawkesMgfConsts& c;
  HawkesMgfConsts d;
  cd phi, h0;              // h0 = (phi + 1) phi / 2 - psi: drift0 = sigma^2 h0
  double dphi;             // Phi: 0 on the ODE directions, -1 on the gamma direction (whose d is zero)
  __device__ __forceinline__ void operator()(const cd (&A)[3], const cd (&dA)[3], cd (&out)[3]) const {
    const cd zp = (phi - c.beta1_p * A[1]) - c.beta1_m * A[2], zm = (phi - c.beta2_p * A[1]) - c.beta2_m * A[2];
    const cd bp = ((c.beta1_p * dA[1] + c.beta1_m * dA[2]) + d.beta1_p * A[1]) + d.beta1_m * A[2];
    const cd bm = ((c.beta2_p * dA[1] + c.beta2_m * dA[2]) + d.beta2_p * A[1]) + d.beta2_m * A[2];
    const cd dzp = Phi ? mk(dphi) - bp : -bp, dzm = Phi ? mk(dphi) - bm : -bm;
    out[0] = (((c.kt_p * dA[1] + c.kt_m * dA[2]) + d.kt_p * A[1]) + d.kt_m * A[2]) + d.sigma2 * h0;
    if (Phi) out[0] = out[0] + (c.sigma2 * dphi) * (phi + mk(0.5));
    out[1] = (hawkes_djump(zp, dzp, c.shift_p, c.mean_p, d.shift_p, d.mean_p) - (c.kappa_p * dA[1] + d.kappa_p * A[1])) + d.comp_p * phi;
    if (Phi) out[1] = out[1] + mk(c.comp_p * dphi);
    out[2] = (hawkes_djump(zm, dzm, c.shift_m, c.mean_m, d.shift_m, d.mean_m) - (c.kappa_m * dA[2] + d.kappa_m * A[2])) + d.comp_m * phi;
    if (Phi) out[2] = out[2] + mk(c.comp_m * dphi);
  }
};

// hawkes_mgf_kernel in forward mode: one thread = one (grid point, direction), the primal integration of hawkes_mgf_kernel (same
// rk45_generic, same mesh) plus one tangent.  The D = 13 ODE directions of a point, and with Phi the gamma direction of the risk kernel
// (DESIGN.md §4.12) as the 14th, are neighbouring threads, so a warp runs few meshes.  restart = 0: A and dA carried over the maturity
// increments dtaus (the grid); restart != 0 (Phi only): every maturity restarts from A = dA = 0 and integrates over its full ttm dtaus[m]
// (the normaliser points, as hawkes_mgf_kernel's restart mode).  Outputs: dlog_mgf [15 + Phi][M][P] (HAWKES_GREEK_PARAMS order, then
// HAWKES_RISK_PREMIA_GREEK_PARAMS' row 15 = d/d gamma; rows 5 / 10 = a_p / a_m), log_mgf [M][P], status [P] (!Phi only), nfev [P] (each
// optional but dlog_mgf).
template <int TPB, bool Phi>
__global__ void __launch_bounds__(TPB) hawkes_mgf_tangent_kernel(const cd* __restrict__ phi, int P, int M, const double* __restrict__ dtaus,
                                                                 HawkesMgfConsts c, HawkesTangentDirs dirs, int restart,
                                                                 cd* __restrict__ dlog_mgf, cd* __restrict__ log_mgf, int* __restrict__ status,
                                                                 int* __restrict__ nfev) {
  constexpr int D = kHawkesOdeDirs + Phi;
  __shared__ cd stage_smem[6 * 3 * TPB];
  __shared__ cd tan_smem[8 * 3 * TPB];
  const int t = blockIdx.x * TPB + threadIdx.x;
  if (t >= P * D) return;
  const int p = t / D, dir = t % D;
  const bool gdir = Phi && dir == kHawkesOdeDirs;
#pragma unroll
  for (int i = 0; i < 18; ++i) stage_smem[threadIdx.x + i * TPB] = mk(0.0);
#pragma unroll
  for (int i = 0; i < 24; ++i) tan_smem[threadIdx.x + i * TPB] = mk(0.0);
  StageStore<3, TPB> K{stage_smem + threadIdx.x};
  const cd ph = phi[p];
  const cd h0 = 0.5 * ((ph + mk(1.0)) * ph);
  const HawkesRhsFn f{c, ph, c.sigma2 * h0};
  const HawkesMgfConsts zero{0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  TangentHook<3, TPB, HawkesTanRhsFn<Phi>> tan{HawkesTanRhsFn<Phi>{c, gdir ? zero : dirs.d[dir], ph, h0, gdir ? -1.0 : 0.0},
                                               {StageStore<3, TPB>{tan_smem + threadIdx.x}, {}}};   // dy = 0
  cd A[3] = {mk(0.0), mk(0.0), mk(0.0)};
  const int row = gdir ? kHawkesGreekParams : hawkes_dir_row(dir);
  int st = 0, nf = 0;
  for (int m = 0; m < M; ++m) {
    if (Phi && restart) {
#pragma unroll
      for (int k = 0; k < 3; ++k) A[k] = tan.t.dy[k] = mk(0.0);
    }
    int nfe = 0;
    st |= rk45_generic<3, TPB>(A, dtaus[m], f, K, &nfe, &tan);
    nf += nfe;
    dlog_mgf[((size_t)row * M + m) * P + p] = (tan.t.dy[0] + tan.t.dy[1] * c.lambda_p) + tan.t.dy[2] * c.lambda_m;
    if (dir == 0) {
      dlog_mgf[((size_t)5 * M + m) * P + p] = A[1];
      dlog_mgf[((size_t)10 * M + m) * P + p] = A[2];
      if (log_mgf) log_mgf[(size_t)m * P + p] = (A[0] + A[1] * c.lambda_p) + A[2] * c.lambda_m;
    }
  }
  if (dir == 0) {
    if (!Phi && status) status[p] = st;
    if (nfev) nfev[p] = nf;
  }
}

// Fourier sums of fourier_vanilla_kernel (|Re phi| = 1/2 branch, real weights w) and their derivatives, one CTA per strike, fixed-order
// block_sum:  S = sum w Re e^z,  S_x = sum w Re(-phi e^z),  S_xx = sum w Re(phi^2 e^z),  S_p = sum w Re(e^z dlm_p),  z = lm - x phi,
// x = ln(F/K); a grid point whose price term is NaN is skipped in every sum.  greeks [2 + NP][J]: delta, gamma, d price / d parameter.
template <int NP>
__global__ void __launch_bounds__(kFourierThreads) fourier_vanilla_greeks_kernel(const cd* __restrict__ log_mgf, const cd* __restrict__ dlog_mgf,
                                                                                const cd* __restrict__ phi, int P, int M,
                                                                                const StrikeSpec* __restrict__ specs, int is_spot,
                                                                                double* __restrict__ greeks) {
  const StrikeSpec sp = specs[blockIdx.x];
  const cd* lm = log_mgf + (size_t)sp.slice * P;
  const double x = log(sp.forward / sp.strike);
  double acc[3 + NP] = {};
  strike_sum(phi, P, acc, [&](int j, double dp, cd ph) {
    const double w = (dp / M_PI) / (ph.im * ph.im + 0.25);
    const cd e = cexp_(lm[j] - x * ph);
    const cd term = mk(w) * e;
    if (term.re == term.re) {
      acc[0] += term.re;
      acc[1] += w * (-(ph * e)).re;
      acc[2] += w * ((ph * ph) * e).re;
#pragma unroll
      for (int k = 0; k < NP; ++k) acc[3 + k] += w * (e * dlog_mgf[((size_t)k * M + sp.slice) * P + j]).re;
    }
  });
  if (threadIdx.x == 0) {
    const double S = acc[0], Sx = acc[1], Sxx = acc[2], F = sp.forward, K = sp.strike, df = sp.discfactor;
    const int J = gridDim.x;
    const bool call = sp.type == B200SV_CALL || sp.type == B200SV_INV_CALL;
    double delta, gamma, scale;
    if (is_spot) {             // C = df (F - K S), P = df (K - K S)
      delta = call ? df * (1.0 - K * Sx / F) : -df * K * Sx / F;
      gamma = -df * K * (Sxx - Sx) / (F * F);
      scale = -df * K;
    } else {                   // C = F df (1 - S), P = df (K - F S)
      delta = call ? df * (1.0 - S - Sx) : -df * (S + Sx);
      gamma = -df * (Sx + Sxx) / F;
      scale = -F * df;
    }
    greeks[blockIdx.x] = delta;
    greeks[J + blockIdx.x] = gamma;
#pragma unroll
    for (int k = 0; k < NP; ++k) greeks[(size_t)(2 + k) * J + blockIdx.x] = scale * acc[3 + k];
  }
}

// ---- Hawkes jump-diffusion under the risk kernel (DESIGN.md §4.12) ----
// risk_premia_gamma moves every transform point, on the grid (Re phi = -1/2 - gamma) and at the two normaliser points (-gamma,
// -gamma - 1), by d phi / d gamma = -1: a 14th tangent direction, in the transform variable, next to the 13 ODE directions (the Phi
// instantiations of HawkesTanRhsFn, hawkes_mgf_tangent_kernel, HawkesTan2RhsFn and hawkes_mgf_hessian_kernel).
constexpr int kHawkesRpParams = kHawkesGreekParams + 1;      // HAWKES_RISK_PREMIA_GREEK_PARAMS: HAWKES_GREEK_PARAMS, then risk_premia_gamma

// Sums of fourier_gamma_batch_kernel (same weight branch, same NaN skip) and their derivatives, one CTA per strike, fixed-order block_sum:
// with e = exp(lm - x phi), x = ln(F/K):  S = sum Re(w e),  S_x = sum Re(-w phi e),  S_xx = sum Re(w phi^2 e),  S_p = sum Re(w e dlm_p),
// and for gamma S_g = sum Re(w e (x + dlm_g)) (the grid moves, phi + gamma does not, so w is fixed).  The prices C = G - n K^(1+g) S,
// P = K - n K^(1+g) S with n = e^{-l0}, G = F e^{l1} n (norm_gfwd [M][2], the pricing route's own) give
//   delta = [C] G / F - n K^(1+g) S_x / F,   gamma = -n K^(1+g) (S_xx - S_x) / F^2,
//   d/dp  = [C] G (l1_p - l0_p) - n K^(1+g) (S_p - l0_p S [+ ln K S for gamma]),
// where l0_p, l1_p = Re dnorm [16][M][2] (the restarted tangents at -gamma, -gamma - 1).  greeks [2 + 16][J].
__global__ void __launch_bounds__(kFourierThreads) fourier_gamma_greeks_kernel(const cd* __restrict__ log_mgf, const cd* __restrict__ dlog_mgf,
                                                                              const cd* __restrict__ dnorm, const cd* __restrict__ phi, int P,
                                                                              int M, const StrikeSpec* __restrict__ specs, double gamma,
                                                                              const double* __restrict__ norm_gfwd, double* __restrict__ greeks) {
  constexpr int NP = kHawkesRpParams;
  const StrikeSpec sp = specs[blockIdx.x];
  const cd* lm = log_mgf + (size_t)sp.slice * P;
  const double x = log(sp.forward / sp.strike);
  const bool fast = fabs(phi[0].re - (0.5 + gamma)) < 1e-10;
  double acc[3 + NP] = {};
  strike_sum(phi, P, acc, [&](int j, double dp, cd ph) {
    const cd pg = ph + mk(gamma);
    const cd w = fast ? mk((dp / M_PI) / (ph.im * ph.im + 0.25)) : -(mk(dp / M_PI) / ((pg + mk(1.0)) * pg));
    const cd e = cexp_(lm[j] - x * ph);
    const cd term = w * e;
    if (term.re == term.re) {
      acc[0] += term.re;
      acc[1] += (w * -(ph * e)).re;
      acc[2] += (w * ((ph * ph) * e)).re;
#pragma unroll
      for (int k = 0; k < NP - 1; ++k) acc[3 + k] += (term * dlog_mgf[((size_t)k * M + sp.slice) * P + j]).re;
      acc[2 + NP] += (term * (mk(x) + dlog_mgf[((size_t)(NP - 1) * M + sp.slice) * P + j])).re;
    }
  });
  if (threadIdx.x == 0) {
    const double S = acc[0], Sx = acc[1], Sxx = acc[2], F = sp.forward, K = sp.strike;
    const double n = norm_gfwd[2 * (size_t)sp.slice], G = norm_gfwd[2 * (size_t)sp.slice + 1], ngk = n * pow(K, 1.0 + gamma);
    const int J = gridDim.x;
    const bool call = sp.type == B200SV_CALL;
    greeks[blockIdx.x] = (call ? G / F : 0.0) - ngk * Sx / F;
    greeks[J + blockIdx.x] = -ngk * (Sxx - Sx) / (F * F);
#pragma unroll
    for (int k = 0; k < NP; ++k) {
      const double l0 = dnorm[((size_t)k * M + sp.slice) * 2].re, l1 = dnorm[((size_t)k * M + sp.slice) * 2 + 1].re;
      const double s = (acc[3 + k] - l0 * S) + (k == NP - 1 ? log(K) * S : 0.0);
      greeks[(size_t)(2 + k) * J + blockIdx.x] = (call ? G * (l1 - l0) : 0.0) - ngk * s;
    }
  }
}

// --------------------------------------------------------------------------------------------------------------------
// Second-order forward-mode sensitivities of the Fourier chain pricers (DESIGN.md §4.4)
// --------------------------------------------------------------------------------------------------------------------
// row of the pair (p, q), p <= q < n, in the row-major upper triangle [n (n + 1) / 2]
__host__ __device__ constexpr int tri_index(int p, int q, int n) { return p * n - p * (p - 1) / 2 + (q - p); }
// the pair of row r of that triangle
__device__ __forceinline__ void tri_pair(int r, int n, int& p, int& q) {
  p = 0;
  while (r >= n - p) r -= n - p++;
  q = p + r;
}

constexpr int kLogsvOdePairs = kLogsvOdeDirs * (kLogsvOdeDirs + 1) / 2;     // 15 pairs over (theta, kappa1, kappa2, beta, volvol)
constexpr int kHestonOdePairs = kHestonOdeDirs * (kHestonOdeDirs + 1) / 2;  // 10 pairs over (theta, kappa, rho, volvol)

// d2(LogsvModel field) / d(direction p) d(direction q) for the kLogsvOdePairs pairs (tri_index order over the ODE directions); the fields
// are polynomials of degree <= 3 in the parameters, kappa2 held fixed when kappa1 or theta moves as in make_model_tangents
static void make_model_hessian(const b200sv_logsv_params& p, double eta, bool spot, LogsvModelTangent (&h)[kLogsvOdePairs]) {
  for (auto& t : h) t = LogsvModelTangent{0, 0, 0, 0, 0, 0, 0, 0, 0};
  const double v2 = p.beta * p.beta + p.volvol * p.volvol, th2 = p.theta * p.theta;
  constexpr int D = kLogsvOdeDirs;
  LogsvModelTangent& tt = h[tri_index(0, 0, D)];     // theta theta
  tt.th2 = 2.0;
  tt.qv2 = 2.0 * v2;
  tt.lam = spot ? 0.0 : 2.0 * p.beta * eta;
  h[tri_index(0, 2, D)].kp = 1.0;                    // theta kappa2
  LogsvModelTangent& tb = h[tri_index(0, 3, D)];     // theta beta
  tb.qv = 2.0 * p.beta;
  tb.qv2 = 4.0 * p.theta * p.beta;
  tb.lam = spot ? 0.0 : 2.0 * p.theta * eta;
  tb.kp = spot ? 0.0 : -2.0 * eta;
  LogsvModelTangent& tv = h[tri_index(0, 4, D)];     // theta volvol
  tv.qv = 2.0 * p.volvol;
  tv.qv2 = 4.0 * p.theta * p.volvol;
  for (int d : {3, 4}) {                             // beta beta, volvol volvol
    LogsvModelTangent& s = h[tri_index(d, d, D)];
    s.v2 = 2.0;
    s.qv = 2.0 * p.theta;
    s.qv2 = 2.0 * th2;
  }
}

// make_coef differentiated twice: linear in the fields except the products th2 b, theta b (b = beta_eta phi) and th2 eta2, theta eta2,
// which take the second-order product rule
__device__ __forceinline__ Coef make_d2coef(const LogsvModel& m, const LogsvModelTangent& dp, const LogsvModelTangent& dq,
                                            const LogsvModelTangent& d2, cd phi, cd psi) {
  Coef c;
  const cd b = m.beta_eta * phi, bp = dp.beta_eta * phi, bq = dq.beta_eta * phi, b2 = d2.beta_eta * phi;
  const cd dtb = ((d2.th2 * b + dp.th2 * bq) + dq.th2 * bp) + m.th2 * b2;          // d2(th2 b)
  const cd d1b = ((d2.theta * b + dp.theta * bq) + dq.theta * bp) + m.theta * b2;  // d2(theta b)
  c.l01 = mk(d2.lam) - dtb;
  c.l11 = mk(-d2.kp) - 2.0 * d1b;
  c.l12 = 2.0 * (mk(d2.lam + d2.qv) - dtb);
  c.l21 = mk(-d2.k2p) - b2;
  c.l22 = mk(d2.v2 - 2.0 * d2.kp) - 4.0 * d1b;
  c.l23 = 3.0 * (mk(2.0 * d2.qv) - dtb);
  c.l32 = -2.0 * (mk(d2.k2p) + b2);
  c.l33 = 3.0 * (mk(d2.v2 - d2.kp) - 2.0 * d1b);
  c.l34 = 4.0 * (mk(3.0 * d2.qv) - dtb);
  c.l43 = -3.0 * (mk(d2.k2p) + b2);
  c.l44 = 2.0 * (mk(d2.v2 - 2.0 * d2.kp) - 4.0 * d1b);
  const cd r = m.spot ? phi * (phi + mk(1.0)) - 2.0 * psi : phi * (phi - mk(1.0)) - 2.0 * psi;
  c.h0 = (0.5 * d2.th2 * m.eta2) * r;
  c.h1 = (d2.theta * m.eta2) * r;
  c.h2 = mk(0.0);
  return c;
}

// the products X_i Y_j + Y_i X_j over the pairs q = {11, 12, 22, 13, 14, 23, 24, 33} of rhs_rows
template <int N>
__device__ __forceinline__ void sym_products(const cd (&X)[N], const cd (&Y)[N], cd (&out)[8]) {
  constexpr int I[8] = {1, 1, 2, 1, 1, 2, 2, 3}, J[8] = {1, 2, 2, 3, 4, 3, 4, 3};
#pragma unroll
  for (int k = 0; k < 8; ++k) out[k] = (I[k] < N && J[k] < N) ? X[I[k]] * Y[J[k]] + Y[I[k]] * X[J[k]] : mk(0.0);
}

// The three right-hand sides of one parameter pair (p, q), f(A) = rows(q(A), A; F) with F = (v2, qv, qv2, Coef):
//   d_p f   = rows(dq_p, dA_p; F) + rows(q, A; F_p, with H)                                  (rhs_tangent), the same for q
//   d_pq f  = rows(d2q, d2A; F) + rows(dq_p, dA_p; F_q) + rows(dq_q, dA_q; F_p) + rows(q, A; F_pq, with H)
// with dq_p = sym(A, dA_p) and d2q = sym(A, d2A) + sym(dA_p, dA_q): J(A) d2A + f_AA(dA_p, dA_q) + d_p J(A) dA_q + d_q J(A) dA_p + d_pq f(A).
template <int N, int TPB>
struct LogsvTan2RhsFn {
  const LogsvModel* m;
  const CoefView<TPB>* c;
  LogsvModelTangent dmp, dmq, d2m;
  CoefView<TPB> dcp, dcq, d2c;
  __device__ __forceinline__ void operator()(const cd (&Y)[N], const cd (&dYp)[N], const cd (&dYq)[N], const cd (&d2Y)[N], cd (&op)[N],
                                             cd (&oq)[N], cd (&opq)[N]) const {
    rhs_tangent<N, TPB>(Y, dYp, *m, *c, dmp, dcp, op);
    rhs_tangent<N, TPB>(Y, dYq, *m, *c, dmq, dcq, oq);
    cd q[8], s[8], t[8], r[N];
    sym_products<N>(Y, d2Y, q);
    sym_products<N>(dYp, dYq, s);
#pragma unroll
    for (int k = 0; k < 8; ++k) q[k] = q[k] + s[k];
    rhs_rows<N, TPB, false>(q, d2Y, m->v2, m->qv, m->qv2, *c, opq);
    sym_products<N>(Y, dYp, s);
    rhs_rows<N, TPB, false>(s, dYp, dmq.v2, dmq.qv, dmq.qv2, dcq, r);
#pragma unroll
    for (int k = 0; k < N; ++k) opq[k] = opq[k] + r[k];
    sym_products<N>(Y, dYq, s);
    rhs_rows<N, TPB, false>(s, dYq, dmp.v2, dmp.qv, dmp.qv2, dcp, r);
#pragma unroll
    for (int k = 0; k < N; ++k) opq[k] = opq[k] + r[k];
#pragma unroll
    for (int k = 0; k < 8; ++k) t[k] = mk(0.0);
    t[0] = Y[1] * Y[1]; t[1] = Y[1] * Y[2]; t[2] = Y[2] * Y[2];
    if constexpr (N == 5) {
      t[3] = Y[1] * Y[3]; t[4] = Y[1] * Y[4]; t[5] = Y[2] * Y[3]; t[6] = Y[2] * Y[4]; t[7] = Y[3] * Y[3];
    }
    rhs_rows<N, TPB, true>(t, Y, d2m.v2, d2m.qv, d2m.qv2, d2c, r);
#pragma unroll
    for (int k = 0; k < N; ++k) opq[k] = opq[k] + r[k];
  }
};

// TangentHook one order higher: the tangents of directions p and q and the mixed second-order tangent of the pair, three TangentStores
// stepped on rk45_generic's attempts.  Tan2Rhs: ``void operator()(Y, dYp, dYq, d2Y, out_p, out_q, out_pq) const``.
template <int N, int TPB, typename Tan2Rhs>
struct Tangent2Hook {
  Tan2Rhs f;
  TangentStore<N, TPB> p, q, pq;

  __device__ __forceinline__ void eval(int s, const cd (&Y)[N], const cd (&dYp)[N], const cd (&dYq)[N], const cd (&d2Y)[N]) {
    cd op[N], oq[N], opq[N];
    f(Y, dYp, dYq, d2Y, op, oq, opq);
#pragma unroll
    for (int k = 0; k < N; ++k) {
      p.dK.at(s, k) = op[k];
      q.dK.at(s, k) = oq[k];
      pq.dK.at(s, k) = opq[k];
    }
  }
  __device__ __forceinline__ void start(const cd (&y)[N]) { eval(0, y, p.dy, q.dy, pq.dy); }
  __device__ __forceinline__ void stage(int s, const cd (&yt)[N], double h) {
    cd a[N], b[N], c[N];
    p.stage_input(s, h, a);
    q.stage_input(s, h, b);
    pq.stage_input(s, h, c);
    eval(s, yt, a, b, c);
  }
  __device__ __forceinline__ void last(const cd (&yn)[N], double h) {
    cd a[N], b[N], c[N];
    p.candidate(h, a);
    q.candidate(h, b);
    pq.candidate(h, c);
    eval(6, yn, a, b, c);
  }
  __device__ __forceinline__ void accept() { accept_tangents<N, TPB>(p, q, pq); }
};

constexpr int kHessianTPB = 8;   // shared memory per thread: 6N primal stages + 3 x 8N tangent stages + 4 x 14 coefficients

// One thread = one (grid point, ODE pair p <= q): the primal integration of logsv_mgf_kernel (same rk45_generic, same mesh) plus the
// tangents of p and q and their mixed second-order tangent.  The 15 pairs of a point are neighbouring threads.  lm = sum_k A_k y^k with
// y = sigma0 - theta gives
//   d2lm_pq = sum_k d2A_k y^k + (dA_p,k y_q + dA_q,k y_p) k y^(k-1) + A_k y_p y_q k (k-1) y^(k-2),   y_sigma0 = 1, y_theta = -1;
// sigma0 has no ODE tangent, so the diagonal thread of direction p also writes the pair (sigma0, p) and pair 0 writes (sigma0, sigma0).
// dspec [M][5], d2spec [M][15]: first and second field derivatives.  Output d2log_mgf [21][M][P] (tri_index over LOGSV_GREEK_PARAMS).
template <int N>
__global__ void __launch_bounds__(kHessianTPB) logsv_mgf_hessian_kernel(const cd* __restrict__ phi, int P, int M, const ChainSpec* __restrict__ spec,
                                                                         const LogsvModelTangent* __restrict__ dspec,
                                                                         const LogsvModelTangent* __restrict__ d2spec, double y,
                                                                         cd* __restrict__ d2log_mgf) {
  constexpr int TPB = kHessianTPB, D = kLogsvOdeDirs, NP = 1 + kLogsvOdeDirs;
  __shared__ cd stage_smem[6 * N * TPB];
  __shared__ cd tan_smem[3 * 8 * N * TPB];
  __shared__ cd coef_smem[4 * 14 * TPB];
  const int t = blockIdx.x * TPB + threadIdx.x;
  if (t >= P * kLogsvOdePairs) return;
  const int p = t / kLogsvOdePairs, pair = t % kLogsvOdePairs;
  int dp, dq;
  tri_pair(pair, D, dp, dq);
#pragma unroll
  for (int i = 0; i < 6 * N; ++i) stage_smem[threadIdx.x + i * TPB] = mk(0.0);
#pragma unroll
  for (int i = 0; i < 3 * 8 * N; ++i) tan_smem[threadIdx.x + i * TPB] = mk(0.0);
  StageStore<N, TPB> K{stage_smem + threadIdx.x};
  const CoefView<TPB> c{coef_smem + threadIdx.x};
  Tangent2Hook<N, TPB, LogsvTan2RhsFn<N, TPB>> tan;
  tan.f.c = &c;
  tan.f.dcp = CoefView<TPB>{coef_smem + 14 * TPB + threadIdx.x};
  tan.f.dcq = CoefView<TPB>{coef_smem + 28 * TPB + threadIdx.x};
  tan.f.d2c = CoefView<TPB>{coef_smem + 42 * TPB + threadIdx.x};
  tan.p.dK = StageStore<N, TPB>{tan_smem + threadIdx.x};
  tan.q.dK = StageStore<N, TPB>{tan_smem + 8 * N * TPB + threadIdx.x};
  tan.pq.dK = StageStore<N, TPB>{tan_smem + 16 * N * TPB + threadIdx.x};
  cd A[N];
#pragma unroll
  for (int k = 0; k < N; ++k) {
    A[k] = mk(0.0);
    tan.p.dy[k] = tan.q.dy[k] = tan.pq.dy[k] = mk(0.0);
  }
  const cd ph = phi[p], ps = mk(0.0);
  const double y2 = y * y;
  const double ys[5] = {1.0, y, y2, y2 * y, y2 * y2};
  const double dys[5] = {0.0, 1.0, 2.0 * y, 3.0 * y2, 4.0 * (y2 * y)};
  const double d2ys[5] = {0.0, 0.0, 2.0, 6.0 * y, 12.0 * y2};
  const double yp = dp == 0 ? -1.0 : 0.0, yq = dq == 0 ? -1.0 : 0.0;
  for (int mm = 0; mm < M; ++mm) {
    const LogsvModel model = spec[mm].model;
    store_coef<TPB>(coef_smem + threadIdx.x, make_coef(model, ph, ps));
    tan.f.m = &model;
    tan.f.dmp = dspec[mm * D + dp];
    tan.f.dmq = dspec[mm * D + dq];
    tan.f.d2m = d2spec[mm * kLogsvOdePairs + pair];
    store_coef<TPB>(coef_smem + 14 * TPB + threadIdx.x, make_dcoef(model, tan.f.dmp, ph, ps));
    store_coef<TPB>(coef_smem + 28 * TPB + threadIdx.x, make_dcoef(model, tan.f.dmq, ph, ps));
    store_coef<TPB>(coef_smem + 42 * TPB + threadIdx.x, make_d2coef(model, tan.f.dmp, tan.f.dmq, tan.f.d2m, ph, ps));
    rk45_generic<N, TPB>(A, spec[mm].dtau, LogsvRhsFn<N, TPB>{model, c}, K, nullptr, &tan);
    cd h = mk(0.0), hs = mk(0.0), hss = mk(0.0);
#pragma unroll
    for (int k = 0; k < N; ++k) {
      h = h + (tan.pq.dy[k] * ys[k] + (tan.p.dy[k] * yq + tan.q.dy[k] * yp) * dys[k] + A[k] * (yp * yq * d2ys[k]));
      hs = hs + (tan.p.dy[k] * dys[k] + A[k] * (yp * d2ys[k]));      // (sigma0, p): y_sigma0 = 1, no ODE tangent
      hss = hss + A[k] * d2ys[k];                                      // (sigma0, sigma0)
    }
    d2log_mgf[((size_t)tri_index(1 + dp, 1 + dq, NP) * M + mm) * P + p] = h;
    if (dp == dq) d2log_mgf[((size_t)tri_index(0, 1 + dp, NP) * M + mm) * P + p] = hs;
    if (pair == 0) d2log_mgf[(size_t)mm * P + p] = hss;
  }
}

// hyper-dual complex numbers (value, derivative in p, derivative in q, mixed second derivative) for the Heston closed form, through the
// same principal csqrt / cexp / clog and Smith division as dcd
struct hcd {
  cd v, d1, d2, d12;
};
__device__ __forceinline__ hcd hmk(cd v) { return hcd{v, mk(0.0), mk(0.0), mk(0.0)}; }
__device__ __forceinline__ hcd operator+(hcd a, hcd b) { return hcd{a.v + b.v, a.d1 + b.d1, a.d2 + b.d2, a.d12 + b.d12}; }
__device__ __forceinline__ hcd operator-(hcd a, hcd b) { return hcd{a.v - b.v, a.d1 - b.d1, a.d2 - b.d2, a.d12 - b.d12}; }
__device__ __forceinline__ hcd operator-(hcd a) { return hcd{-a.v, -a.d1, -a.d2, -a.d12}; }
__device__ __forceinline__ hcd operator*(double s, hcd a) { return hcd{s * a.v, s * a.d1, s * a.d2, s * a.d12}; }
__device__ __forceinline__ hcd operator*(hcd a, hcd b) {
  return hcd{a.v * b.v, a.d1 * b.v + a.v * b.d1, a.d2 * b.v + a.v * b.d2, ((a.d12 * b.v + a.d1 * b.d2) + a.d2 * b.d1) + a.v * b.d12};
}
__device__ __forceinline__ hcd operator/(hcd a, hcd b) {   // q = a / b from a = q b differentiated
  const cd q = a.v / b.v, q1 = (a.d1 - q * b.d1) / b.v, q2 = (a.d2 - q * b.d2) / b.v;
  return hcd{q, q1, q2, (((a.d12 - q1 * b.d2) - q2 * b.d1) - q * b.d12) / b.v};
}
__device__ __forceinline__ hcd sqrt_(hcd z) {              // s^2 = z differentiated
  const cd s = sqrt_(z.v), s1 = z.d1 / (2.0 * s), s2 = z.d2 / (2.0 * s);
  return hcd{s, s1, s2, (z.d12 - 2.0 * (s1 * s2)) / (2.0 * s)};
}
__device__ __forceinline__ hcd exp_(hcd z) {
  const cd e = exp_(z.v);
  return hcd{e, e * z.d1, e * z.d2, e * (z.d12 + z.d1 * z.d2)};
}
__device__ __forceinline__ hcd log_(hcd z) {
  const cd l1 = z.d1 / z.v, l2 = z.d2 / z.v;
  return hcd{log_(z.v), l1, l2, (z.d12 - l1 * z.d2) / z.v};
}

// heston_mgf_kernel in second-order forward mode: one thread = one (grid point, pair p <= q of theta | kappa | rho | volvol), (a, b) as
// hyper-dual numbers carried over the maturities.  log_mgf = a + b v0, so d2/dv0^2 = 0 and d2/dv0 dq = db/dq: the diagonal thread of q
// writes the latter, pair 0 the former.  d2log_mgf [15][M][P] (tri_index over HESTON_GREEK_PARAMS).
__global__ void heston_mgf_hessian_kernel(const cd* __restrict__ phi, int P, int M, const double* __restrict__ dtaus, b200sv_heston_params hp,
                                          cd* __restrict__ d2log_mgf) {
  constexpr int D = kHestonOdeDirs, NP = 1 + kHestonOdeDirs;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= P * kHestonOdePairs) return;
  const int p = t / kHestonOdePairs, pair = t % kHestonOdePairs;
  int dp, dq;
  tri_pair(pair, D, dp, dq);
  const double x[D] = {hp.theta, hp.kappa, hp.rho, hp.volvol};
  hcd par[D];
#pragma unroll
  for (int k = 0; k < D; ++k) par[k] = hcd{mk(x[k]), mk(k == dp ? 1.0 : 0.0), mk(k == dq ? 1.0 : 0.0), mk(0.0)};
  const HestonClosedForm<hcd, hcd> cf(par[0], par[1], par[2], par[3], phi[p], mk(0.0));
  hcd a = hmk(mk(0.0)), b = hmk(mk(0.0));
  for (int mm = 0; mm < M; ++mm) {
    cf.step(dtaus[mm], a, b);
    d2log_mgf[((size_t)tri_index(1 + dp, 1 + dq, NP) * M + mm) * P + p] = a.d12 + b.d12 * hp.v0;
    if (dp == dq) d2log_mgf[((size_t)tri_index(0, 1 + dp, NP) * M + mm) * P + p] = b.d1;
    if (pair == 0) d2log_mgf[(size_t)mm * P + p] = mk(0.0);
  }
}

// The second-order Fourier sums next to fourier_vanilla_greeks_kernel's, one CTA per strike, fixed-order block_sum:
//   S_p = sum w Re(e^z dlm_p),  S_xp = sum w Re(-phi e^z dlm_p),  S_pq = sum w Re(e^z (d2lm_pq + dlm_p dlm_q)),
// z = lm - x phi, the same NaN-skipping.  Spot: vanna_p = -df K S_xp / F, hessian_pq = -df K S_pq;
// inverse: vanna_p = -df (S_p + S_xp), hessian_pq = -F df S_pq.  vanna [NP][J], hessian [NP (NP + 1) / 2][J] (tri_index rows).
template <int NP>
__global__ void __launch_bounds__(kFourierThreads) fourier_vanilla_hessian_kernel(const cd* __restrict__ log_mgf, const cd* __restrict__ dlog_mgf,
                                                                                 const cd* __restrict__ d2log_mgf, const cd* __restrict__ phi,
                                                                                 int P, int M, const StrikeSpec* __restrict__ specs,
                                                                                 int is_spot, double* __restrict__ vanna,
                                                                                 double* __restrict__ hessian) {
  constexpr int NH = NP * (NP + 1) / 2;
  const StrikeSpec sp = specs[blockIdx.x];
  const cd* lm = log_mgf + (size_t)sp.slice * P;
  const double x = log(sp.forward / sp.strike);
  double acc[2 * NP + NH] = {};
  strike_sum(phi, P, acc, [&](int j, double dp, cd ph) {
    const double w = (dp / M_PI) / (ph.im * ph.im + 0.25);
    const cd e = cexp_(lm[j] - x * ph);
    const cd term = mk(w) * e;
    if (term.re == term.re) {
      cd dl[NP];
#pragma unroll
      for (int k = 0; k < NP; ++k) {
        dl[k] = dlog_mgf[((size_t)k * M + sp.slice) * P + j];
        const cd ed = e * dl[k];
        acc[k] += w * ed.re;
        acc[NP + k] += w * (-(ph * ed)).re;
      }
      int r = 0;
#pragma unroll
      for (int p = 0; p < NP; ++p)
#pragma unroll
        for (int q = p; q < NP; ++q, ++r) acc[2 * NP + r] += w * (e * (d2log_mgf[((size_t)r * M + sp.slice) * P + j] + dl[p] * dl[q])).re;
    }
  });
  if (threadIdx.x == 0) {
    const double F = sp.forward, K = sp.strike, df = sp.discfactor;
    const int J = gridDim.x;
#pragma unroll
    for (int k = 0; k < NP; ++k)
      vanna[(size_t)k * J + blockIdx.x] = is_spot ? -df * K * acc[NP + k] / F : -df * (acc[k] + acc[NP + k]);
    const double scale = is_spot ? -df * K : -F * df;
#pragma unroll
    for (int r = 0; r < NH; ++r) hessian[(size_t)r * J + blockIdx.x] = scale * acc[2 * NP + r];
  }
}

// fourier_vanilla_hessian_kernel for many parameters: at NP = 15 its 2NP + NP(NP+1)/2 = 150 sums per thread do not stay in registers, so
// a strike's rows are split over the CTAs blockIdx.y = 0 .. NH / NP, every CTA recomputing e^z.  blockIdx.y = 0: the 2NP vanna sums S_p,
// S_xp; blockIdx.y = c > 0: the NP Hessian rows [(c - 1) NP, c NP).  Each row is the same fixed-order block_sum, NaN-skipping and
// assembly as there.
template <int NP>
__global__ void __launch_bounds__(kFourierThreads) fourier_vanilla_hessian_split_kernel(const cd* __restrict__ log_mgf,
                                                                                       const cd* __restrict__ dlog_mgf,
                                                                                       const cd* __restrict__ d2log_mgf,
                                                                                       const cd* __restrict__ phi, int P, int M,
                                                                                       const StrikeSpec* __restrict__ specs, int is_spot,
                                                                                       double* __restrict__ vanna, double* __restrict__ hessian) {
  constexpr int NH = NP * (NP + 1) / 2, R = NP;       // Hessian rows per CTA
  const StrikeSpec sp = specs[blockIdx.x];
  const cd* lm = log_mgf + (size_t)sp.slice * P;
  const double x = log(sp.forward / sp.strike);
  const size_t rs = (size_t)M * P;                     // the row stride of dlog_mgf / d2log_mgf
  const cd* dl = dlog_mgf + (size_t)sp.slice * P;
  const cd* d2l = d2log_mgf + (size_t)sp.slice * P;
  const bool vanna_rows = blockIdx.y == 0;
  const int r0 = vanna_rows ? 0 : ((int)blockIdx.y - 1) * R;
  int p0 = 0, q0 = 0;
  if (!vanna_rows) tri_pair(r0, NP, p0, q0);
  double acc[2 * NP] = {};
  strike_sum(phi, P, acc, [&](int j, double dp, cd ph) {
    const double w = (dp / M_PI) / (ph.im * ph.im + 0.25);
    const cd e = cexp_(lm[j] - x * ph);
    const cd term = mk(w) * e;
    if (term.re == term.re) {
      if (vanna_rows) {
#pragma unroll
        for (int k = 0; k < NP; ++k) {
          const cd ed = e * dl[k * rs + j];
          acc[k] += w * ed.re;
          acc[NP + k] += w * (-(ph * ed)).re;
        }
      } else {
        int p = p0, q = q0;
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const int r = r0 + i;
          if (r < NH) acc[i] += w * (e * (d2l[r * rs + j] + dl[p * rs + j] * dl[q * rs + j])).re;
          if (++q == NP) q = ++p;
        }
      }
    }
  });
  if (threadIdx.x == 0) {
    const double F = sp.forward, K = sp.strike, df = sp.discfactor;
    const int J = gridDim.x;
    if (vanna_rows) {
#pragma unroll
      for (int k = 0; k < NP; ++k) vanna[(size_t)k * J + blockIdx.x] = is_spot ? -df * K * acc[NP + k] / F : -df * (acc[k] + acc[NP + k]);
    } else {
      const double scale = is_spot ? -df * K : -F * df;
#pragma unroll
      for (int i = 0; i < R; ++i)
        if (r0 + i < NH) hessian[(size_t)(r0 + i) * J + blockIdx.x] = scale * acc[i];
    }
  }
}

// ---- Hawkes jump-diffusion, second order (DESIGN.md §4.5) ----
// d2(HawkesMgfConsts field) / d(direction p) d(direction q) for the D (D + 1) / 2 pairs of the D directions of hawkes_mgf_hessian_kernel
// (tri_index order over the ODE directions of make_hawkes_tangents, then with D = 14 the transform variable, which no field depends on).
// Nonzero: sigma2 = sigma^2, kt = kappa theta and comp = e^shift / (1 - mean) - 1.
static std::vector<HawkesMgfConsts> make_hawkes_hessian(const b200sv_hawkes_params& p, int D) {
  std::vector<HawkesMgfConsts> h((size_t)D * (D + 1) / 2, HawkesMgfConsts{0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0});
  const double ep = std::exp(p.shift_p) / (1.0 - p.mean_p), em = std::exp(p.shift_m) / (1.0 - p.mean_m);
  h[tri_index(0, 0, D)].sigma2 = 2.0;                                                  // sigma sigma
  h[tri_index(5, 6, D)].kt_p = 1.0;                                                    // theta_p kappa_p
  h[tri_index(9, 10, D)].kt_m = 1.0;                                                   // theta_m kappa_m
  h[tri_index(1, 1, D)].comp_p = ep;                                                   // shift_p shift_p
  h[tri_index(1, 2, D)].comp_p = ep / (1.0 - p.mean_p);                                // shift_p mean_p
  h[tri_index(2, 2, D)].comp_p = 2.0 * ep / ((1.0 - p.mean_p) * (1.0 - p.mean_p));     // mean_p mean_p
  h[tri_index(3, 3, D)].comp_m = em;                                                   // shift_m shift_m
  h[tri_index(3, 4, D)].comp_m = em / (1.0 - p.mean_m);                                // shift_m mean_m
  h[tri_index(4, 4, D)].comp_m = 2.0 * em / ((1.0 - p.mean_m) * (1.0 - p.mean_m));     // mean_m mean_m
  return h;
}

// The three right-hand sides of one pair (p, q) in one hyper-dual evaluation of HawkesRhsFn's arithmetic: with A_k = (A, dA_p, dA_q,
// d2A_pq) and every HawkesMgfConsts field f = (f, df/dp, df/dq, d2f/dp dq), the parts .d1 / .d2 are the tangent right-hand sides
// J(A) dA_p + d_p f(A) (HawkesTanRhsFn) and J(A) dA_q + d_q f(A), and .d12 is
//   J(A) d2A + f_AA(dA_p, dA_q) + d_p J(A) dA_q + d_q J(A) dA_p + d_pq f(A).
// The jump-size MGF E(z; s, m) = e^{-s z} / (1 + m z) goes through hcd's exp_ and Smith division jointly in (z, s, m); the constant -1 of
// E - 1 has no derivative and is left out.  phi = (phi, dphi_p, dphi_q, 0): without Phi, hmk(phi), and h0 comes precomputed.  Phi puts the
// transform variable among the seeded variables (the risk kernel, DESIGN.md §4.13): dphi = -1 on the gamma direction and 0 on the ODE
// directions, so the hyper-dual algebra also forms every phi cross term (h0 = (phi + 1) phi / 2, comp phi and z = phi - beta a inside the
// jump MGFs).  phi is linear in gamma: its own second part is zero.
template <bool Phi>
struct HawkesTan2RhsFn {
  const HawkesMgfConsts& c;
  HawkesMgfConsts dp, dq, d2;
  hcd phi;
  cd h0;                   // !Phi: h0 = (phi + 1) phi / 2 - psi: drift0 = sigma^2 h0
  __device__ __forceinline__ hcd k(double HawkesMgfConsts::*f) const { return hcd{mk(c.*f), mk(dp.*f), mk(dq.*f), mk(d2.*f)}; }
  __device__ __forceinline__ void operator()(const cd (&Y)[3], const cd (&dYp)[3], const cd (&dYq)[3], const cd (&d2Y)[3], cd (&op)[3],
                                             cd (&oq)[3], cd (&opq)[3]) const {
    using H = HawkesMgfConsts;
    const hcd a1{Y[1], dYp[1], dYq[1], d2Y[1]}, a2{Y[2], dYp[2], dYq[2], d2Y[2]}, one = hmk(mk(1.0));
    const hcd zp = (phi - k(&H::beta1_p) * a1) - k(&H::beta1_m) * a2, zm = (phi - k(&H::beta2_p) * a1) - k(&H::beta2_m) * a2;
    const hcd jp = exp_(-(k(&H::shift_p) * zp)) / (one + k(&H::mean_p) * zp);
    const hcd jm = exp_(-(k(&H::shift_m) * zm)) / (one + k(&H::mean_m) * zm);
    const hcd h = Phi ? 0.5 * ((phi + one) * phi) : hmk(h0);
    const hcd o[3] = {(k(&H::kt_p) * a1 + k(&H::kt_m) * a2) + k(&H::sigma2) * h, (jp - k(&H::kappa_p) * a1) + k(&H::comp_p) * phi,
                      (jm - k(&H::kappa_m) * a2) + k(&H::comp_m) * phi};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      op[i] = o[i].d1;
      oq[i] = o[i].d2;
      opq[i] = o[i].d12;
    }
  }
};

constexpr int kHawkesHessianTPB = 32;   // static shared memory per thread: 6 x 3 primal + 3 x 8 x 3 tangent stages = 1 440 B, 45 KB per CTA

// One thread = one (grid point, pair p <= q of the D = 13 ODE directions, with Phi also the gamma direction of hawkes_mgf_tangent_kernel):
// the primal integration of hawkes_mgf_kernel (same rk45_generic, same mesh) plus the tangents of p and q and their mixed second-order
// tangent (Tangent2Hook).  The D (D + 1) / 2 pairs of a point are neighbouring threads.  restart = 0: carried over the maturity increments
// dtaus like A (the grid); restart != 0 (Phi only): every maturity restarts from A = 0 and integrates over its full ttm dtaus[m] (the
// normaliser points).  lm = a0 + a_p lambda_p + a_m lambda_m is linear in the lambdas and they have no ODE tangent, so
//   d2lm_pq = d2a0 + d2a_p lambda_p + d2a_m lambda_m,  d2lm / dlambda_p dq = da_p / dq,  d2lm / dlambda_m dq = da_m / dq,  d2lm / dlambda dlambda = 0:
// the diagonal thread of direction d also writes (lambda_p, d) and (lambda_m, d) (for the phi direction da / dgamma = -da / dphi), pair 0
// the three lambda-lambda rows.  dirs: the first field derivatives (make_hawkes_tangents), d2c [D (D + 1) / 2]: the second
// (make_hawkes_hessian).  Output d2log_mgf [NP (NP + 1) / 2][M][P] (tri_index over HAWKES_GREEK_PARAMS, NP = 15, or with Phi over
// HAWKES_RISK_PREMIA_GREEK_PARAMS, NP = 16).
template <bool Phi>
__global__ void __launch_bounds__(kHawkesHessianTPB) hawkes_mgf_hessian_kernel(const cd* __restrict__ phi, int P, int M,
                                                                               const double* __restrict__ dtaus, HawkesMgfConsts c,
                                                                               HawkesTangentDirs dirs, const HawkesMgfConsts* __restrict__ d2c,
                                                                               int restart, cd* __restrict__ d2log_mgf) {
  constexpr int TPB = kHawkesHessianTPB, D = kHawkesOdeDirs + Phi, NP = kHawkesGreekParams + Phi, NPAIRS = D * (D + 1) / 2;
  __shared__ cd stage_smem[6 * 3 * TPB];
  __shared__ cd tan_smem[3 * 8 * 3 * TPB];
  const int t = blockIdx.x * TPB + threadIdx.x;
  if (t >= P * NPAIRS) return;
  const int p = t / NPAIRS, pair = t % NPAIRS;
  int dp, dq;
  tri_pair(pair, D, dp, dq);
#pragma unroll
  for (int i = 0; i < 18; ++i) stage_smem[threadIdx.x + i * TPB] = mk(0.0);
#pragma unroll
  for (int i = 0; i < 72; ++i) tan_smem[threadIdx.x + i * TPB] = mk(0.0);
  StageStore<3, TPB> K{stage_smem + threadIdx.x};
  const cd ph = phi[p];
  const cd h0 = 0.5 * ((ph + mk(1.0)) * ph);
  const HawkesRhsFn f{c, ph, c.sigma2 * h0};
  const HawkesMgfConsts zero{0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  const bool gp = Phi && dp == kHawkesOdeDirs, gq = Phi && dq == kHawkesOdeDirs;
  const hcd hph{ph, mk(gp ? -1.0 : 0.0), mk(gq ? -1.0 : 0.0), mk(0.0)};
  Tangent2Hook<3, TPB, HawkesTan2RhsFn<Phi>> tan{HawkesTan2RhsFn<Phi>{c, gp ? zero : dirs.d[dp], gq ? zero : dirs.d[dq], d2c[pair], hph, h0},
                                                 {StageStore<3, TPB>{tan_smem + threadIdx.x}, {}},
                                                 {StageStore<3, TPB>{tan_smem + 24 * TPB + threadIdx.x}, {}},
                                                 {StageStore<3, TPB>{tan_smem + 48 * TPB + threadIdx.x}, {}}};   // dy = 0
  cd A[3] = {mk(0.0), mk(0.0), mk(0.0)};
  const int rp = gp ? kHawkesGreekParams : hawkes_dir_row(dp), rq = gq ? kHawkesGreekParams : hawkes_dir_row(dq);
  for (int m = 0; m < M; ++m) {
    if (Phi && restart) {
#pragma unroll
      for (int k = 0; k < 3; ++k) A[k] = tan.p.dy[k] = tan.q.dy[k] = tan.pq.dy[k] = mk(0.0);
    }
    rk45_generic<3, TPB>(A, dtaus[m], f, K, nullptr, &tan);
    d2log_mgf[((size_t)tri_index(rp, rq, NP) * M + m) * P + p] = (tan.pq.dy[0] + tan.pq.dy[1] * c.lambda_p) + tan.pq.dy[2] * c.lambda_m;
    if (dp == dq) {
      d2log_mgf[((size_t)tri_index(min(5, rp), max(5, rp), NP) * M + m) * P + p] = tan.p.dy[1];
      d2log_mgf[((size_t)tri_index(min(10, rp), max(10, rp), NP) * M + m) * P + p] = tan.p.dy[2];
    }
    if (pair == 0) {
      d2log_mgf[((size_t)tri_index(5, 5, NP) * M + m) * P + p] = mk(0.0);
      d2log_mgf[((size_t)tri_index(5, 10, NP) * M + m) * P + p] = mk(0.0);
      d2log_mgf[((size_t)tri_index(10, 10, NP) * M + m) * P + p] = mk(0.0);
    }
  }
}

// ---- Hawkes jump-diffusion under the risk kernel, second order (DESIGN.md §4.13) ----
// The second-order risk-kernel sums next to fourier_gamma_greeks_kernel's (same weight branch, same NaN skip, fixed-order block_sum), a
// strike split over the CTAs blockIdx.y as in fourier_vanilla_hessian_split_kernel.  With e = exp(lm - x phi), x = ln(F/K), the per-strike
// tangents T_p = dlm_p (T_gamma = dlm_gamma + x) and T_pq = d2lm_pq:
//   S = sum Re(w e),  S_x = sum Re(-w phi e),  S_p = sum Re(w e T_p),  S_xp = sum Re(w e (-phi T_p + [p = gamma])),
//   S_pq = sum Re(w e (T_p T_q + T_pq)).
// blockIdx.y = 0: S, S_x, S_p, S_xp and vanna_p = ([C] G g_p - c (S_xp + c_p S_x)) / F;  blockIdx.y = b > 0: S, S_p and the Hessian rows
// [(b - 1) NP, b NP):  hessian_pq = [C] G (g_p g_q + g_pq) - c (S_pq + c_p S_q + c_q S_p + (c_p c_q + c_pq) S),  with c = n K^(1+gamma),
// g = l1 - l0, c_p = -l0_p [+ ln K for gamma], c_pq = -l0_pq; l0 / l1 the normaliser log-MGFs (Re dnorm [16][M][2], Re d2norm [136][M][2])
// and (n, G) = norm_gfwd [M][2], the pricing route's own.  vanna [16][J], hessian [136][J] (tri_index rows).
__global__ void __launch_bounds__(kFourierThreads) fourier_gamma_hessian_kernel(const cd* __restrict__ log_mgf, const cd* __restrict__ dlog_mgf,
                                                                               const cd* __restrict__ d2log_mgf, const cd* __restrict__ dnorm,
                                                                               const cd* __restrict__ d2norm, const cd* __restrict__ phi,
                                                                               int P, int M, const StrikeSpec* __restrict__ specs,
                                                                               double gamma, const double* __restrict__ norm_gfwd,
                                                                               double* __restrict__ vanna, double* __restrict__ hessian) {
  constexpr int NP = kHawkesRpParams, NH = NP * (NP + 1) / 2, R = NP;     // Hessian rows per CTA
  const StrikeSpec sp = specs[blockIdx.x];
  const cd* lm = log_mgf + (size_t)sp.slice * P;
  const double x = log(sp.forward / sp.strike);
  const size_t rs = (size_t)M * P;                                         // the row stride of dlog_mgf / d2log_mgf
  const cd* dl = dlog_mgf + (size_t)sp.slice * P;
  const cd* d2l = d2log_mgf + (size_t)sp.slice * P;
  const bool fast = fabs(phi[0].re - (0.5 + gamma)) < 1e-10;
  const bool vanna_rows = blockIdx.y == 0;
  const int r0 = vanna_rows ? 0 : ((int)blockIdx.y - 1) * R;
  int p0 = 0, q0 = 0;
  if (!vanna_rows) tri_pair(r0, NP, p0, q0);
  // acc: S, S_x | S_p [NP] | the vanna CTA's S_xp [NP] or a Hessian CTA's S_pq [R]
  double acc[2 + 2 * NP] = {};
  strike_sum(phi, P, acc, [&](int j, double dp, cd ph) {
    const cd pg = ph + mk(gamma);
    const cd w = fast ? mk((dp / M_PI) / (ph.im * ph.im + 0.25)) : -(mk(dp / M_PI) / ((pg + mk(1.0)) * pg));
    const cd e = cexp_(lm[j] - x * ph);
    const cd term = w * e;
    if (term.re == term.re) {
      const auto T = [&](int k) {
        const cd v = dl[k * rs + j];
        return k == NP - 1 ? v + mk(x) : v;
      };
      acc[0] += term.re;
#pragma unroll
      for (int k = 0; k < NP; ++k) acc[2 + k] += (term * T(k)).re;
      if (vanna_rows) {
        acc[1] += (w * -(ph * e)).re;
#pragma unroll
        for (int k = 0; k < NP; ++k) acc[2 + NP + k] += (term * (k == NP - 1 ? mk(1.0) - ph * T(k) : -(ph * T(k)))).re;
      } else {
        int p = p0, q = q0;
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const int r = r0 + i;
          if (r < NH) acc[2 + NP + i] += (term * (T(p) * T(q) + d2l[r * rs + j])).re;
          if (++q == NP) q = ++p;
        }
      }
    }
  });
  if (threadIdx.x == 0) {
    const double S = acc[0], F = sp.forward, K = sp.strike;
    const double n = norm_gfwd[2 * (size_t)sp.slice], G = norm_gfwd[2 * (size_t)sp.slice + 1], ngk = n * pow(K, 1.0 + gamma);
    const int J = gridDim.x;
    const bool call = sp.type == B200SV_CALL;
    const auto l0 = [&](const cd* v, int r) { return v[((size_t)r * M + sp.slice) * 2].re; };
    const auto l1 = [&](const cd* v, int r) { return v[((size_t)r * M + sp.slice) * 2 + 1].re; };
    const auto cp = [&](int k) { return -l0(dnorm, k) + (k == NP - 1 ? log(K) : 0.0); };
    if (vanna_rows) {
#pragma unroll
      for (int k = 0; k < NP; ++k)
        vanna[(size_t)k * J + blockIdx.x] = ((call ? G * (l1(dnorm, k) - l0(dnorm, k)) : 0.0) - ngk * (acc[2 + NP + k] + cp(k) * acc[1])) / F;
    } else {
      __shared__ double Sp[NP];             // S_p by a run-time index, without moving acc to local memory
#pragma unroll
      for (int k = 0; k < NP; ++k) Sp[k] = acc[2 + k];
      int p = p0, q = q0;
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const int r = r0 + i;
        if (r < NH) {
          const double gp = l1(dnorm, p) - l0(dnorm, p), gq = l1(dnorm, q) - l0(dnorm, q), gpq = l1(d2norm, r) - l0(d2norm, r);
          const double cpp = cp(p), cqq = cp(q), cpq = -l0(d2norm, r);
          hessian[(size_t)r * J + blockIdx.x] = (call ? G * (gp * gq + gpq) : 0.0) -
                                                ngk * (((acc[2 + NP + i] + cpp * Sp[q]) + cqq * Sp[p]) + (cpp * cqq + cpq) * S);
        }
        if (++q == NP) q = ++p;
      }
    }
  }
}

// --------------------------------------------------------------------------------------------------------------------
// Theta of the Fourier chain pricers (DESIGN.md §4.8): d log_mgf / d T_m with the accepted mesh t_0 < ... < t_{K-1} of slice m held and
// only its last step h_K = T_m - t_{K-1} moving (dh_K / dT_m = 1); earlier maturities, the backbone and the grid are held.
// --------------------------------------------------------------------------------------------------------------------
// The derivative of one Dormand-Prince step in its length h at a fixed start y:  G_s = k_s + h dk_s,  dY_s = sum_{j<s} a_sj G_j,
// dk_s = J(Y_s) dY_s (dk_0 = 0),  dy = sum_j b_j G_j.  It is formed on every attempt of rk45_generic and an accepted attempt commits it, so
// after the solve dy is the last accepted step's.  Jvp: ``void operator()(const cd (&Y)[N], const cd (&dY)[N], cd (&out)[N]) const`` =
// J(Y) dY (LogsvJvpFn, or HawkesTanRhsFn with zero constant derivatives).  G in shared memory: stage s holds dk_s until stage s + 1 turns
// it into G_s; stage 6 parks the candidate dy until the acceptance.
template <int N, int TPB, typename Jvp>
struct ThetaHook {
  Jvp f;
  StageStore<N, TPB> K, G;     // K: rk45_generic's own stage store (read only)
  cd dy[N];

  __device__ __forceinline__ void finish_stage(int s, double h) {      // dk_s -> G_s = k_s + h dk_s
#pragma unroll
    for (int k = 0; k < N; ++k) G.at(s, k) = K.at(s, k) + h * G.at(s, k);
  }
  __device__ __forceinline__ void start(const cd (&)[N]) {}
  __device__ __forceinline__ void stage(int s, const cd (&yt)[N], double h) {
    if (s == 1) {
#pragma unroll
      for (int k = 0; k < N; ++k) G.at(0, k) = K.at(0, k);           // G_0 = k_0
    } else {
      finish_stage(s - 1, h);
    }
    cd dyt[N], o[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      cd acc = G.at(0, k) * c_A[s][0];
#pragma unroll
      for (int jj = 1; jj < 5; ++jj) acc = acc + G.at(jj, k) * c_A[s][jj];
      dyt[k] = acc;
    }
    f(yt, dyt, o);
#pragma unroll
    for (int k = 0; k < N; ++k) G.at(s, k) = o[k];
  }
  __device__ __forceinline__ void last(const cd (&)[N], double h) {
    constexpr double B[6] = {35.0 / 384, 0, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84};
    finish_stage(5, h);
#pragma unroll
    for (int k = 0; k < N; ++k) {
      cd acc = G.at(0, k) * B[0];
#pragma unroll
      for (int jj = 2; jj < 6; ++jj) acc = acc + G.at(jj, k) * B[jj];
      G.at(6, k) = acc;
    }
  }
  __device__ __forceinline__ void accept() {
#pragma unroll
    for (int k = 0; k < N; ++k) dy[k] = G.at(6, k);
  }
};

// J(A) dA of the LogSV coefficient ODEs: the Jacobian half of rhs_tangent
template <int N, int TPB>
struct LogsvJvpFn {
  const LogsvModel* m;
  const CoefView<TPB>* c;
  __device__ __forceinline__ void operator()(const cd (&Y)[N], const cd (&dY)[N], cd (&out)[N]) const {
    cd dq[8];
    sym_products<N>(Y, dY, dq);
    rhs_rows<N, TPB, false>(dq, dY, m->v2, m->qv, m->qv2, *c, out);
  }
};

constexpr int kThetaTPB = 8;        // one thread per grid point: 1000 points spread over 125 SMs

// One thread = one grid point: the primal integration of logsv_mgf_kernel (same rk45_generic, same mesh: nfev [P] shows it) plus the theta
// tangent, reset at every slice.  Output dlog_mgf_theta [M][P] = sum_k dA_k y^k.
template <int N>
__global__ void __launch_bounds__(kThetaTPB) logsv_mgf_theta_kernel(const cd* __restrict__ phi, int P, int M, const ChainSpec* __restrict__ spec,
                                                                     double y, cd* __restrict__ dlog_mgf_theta, int* __restrict__ nfev) {
  constexpr int TPB = kThetaTPB;
  __shared__ cd stage_smem[6 * N * TPB];
  __shared__ cd g_smem[7 * N * TPB];
  __shared__ cd coef_smem[14 * TPB];
  const int p = blockIdx.x * TPB + threadIdx.x;
  if (p >= P) return;
#pragma unroll
  for (int i = 0; i < 6 * N; ++i) stage_smem[threadIdx.x + i * TPB] = mk(0.0);
#pragma unroll
  for (int i = 0; i < 7 * N; ++i) g_smem[threadIdx.x + i * TPB] = mk(0.0);
  StageStore<N, TPB> K{stage_smem + threadIdx.x};
  const CoefView<TPB> c{coef_smem + threadIdx.x};
  ThetaHook<N, TPB, LogsvJvpFn<N, TPB>> tan{LogsvJvpFn<N, TPB>{nullptr, &c}, K, StageStore<N, TPB>{g_smem + threadIdx.x}, {}};
  cd A[N];
#pragma unroll
  for (int k = 0; k < N; ++k) A[k] = mk(0.0);
  const cd ph = phi[p], ps = mk(0.0);
  const double y2 = y * y;
  const double ys[5] = {1.0, y, y2, y2 * y, y2 * y2};
  int nf = 0;
  for (int mm = 0; mm < M; ++mm) {
    const LogsvModel model = spec[mm].model;
    store_coef<TPB>(coef_smem + threadIdx.x, make_coef(model, ph, ps));
    tan.f.m = &model;
#pragma unroll
    for (int k = 0; k < N; ++k) tan.dy[k] = mk(0.0);
    int nfe = 0;
    rk45_generic<N, TPB>(A, spec[mm].dtau, LogsvRhsFn<N, TPB>{model, c}, K, &nfe, &tan);
    nf += nfe;
    cd dlm = mk(0.0);
#pragma unroll
    for (int k = 0; k < N; ++k) dlm = dlm + tan.dy[k] * ys[k];
    dlog_mgf_theta[(size_t)mm * P + p] = dlm;
  }
  if (nfev) nfev[p] = nf;
}

// The Hawkes twin: the primal of hawkes_mgf_kernel plus the theta tangent; dlog_mgf_theta [M][P] = da0 + da_p lambda_p + da_m lambda_m.
__global__ void __launch_bounds__(kThetaTPB) hawkes_mgf_theta_kernel(const cd* __restrict__ phi, int P, int M, const double* __restrict__ dtaus,
                                                                    HawkesMgfConsts c, cd* __restrict__ dlog_mgf_theta, int* __restrict__ nfev) {
  constexpr int TPB = kThetaTPB;
  __shared__ cd stage_smem[6 * 3 * TPB];
  __shared__ cd g_smem[7 * 3 * TPB];
  const int p = blockIdx.x * TPB + threadIdx.x;
  if (p >= P) return;
#pragma unroll
  for (int i = 0; i < 18; ++i) stage_smem[threadIdx.x + i * TPB] = mk(0.0);
#pragma unroll
  for (int i = 0; i < 21; ++i) g_smem[threadIdx.x + i * TPB] = mk(0.0);
  StageStore<3, TPB> K{stage_smem + threadIdx.x};
  const cd ph = phi[p];
  const cd h0 = 0.5 * ((ph + mk(1.0)) * ph);
  const HawkesRhsFn f{c, ph, c.sigma2 * h0};
  const HawkesMgfConsts zero{0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};      // no explicit d/dT of the right-hand side
  ThetaHook<3, TPB, HawkesTanRhsFn<false>> tan{HawkesTanRhsFn<false>{c, zero, ph, h0}, K, StageStore<3, TPB>{g_smem + threadIdx.x}, {}};
  cd A[3] = {mk(0.0), mk(0.0), mk(0.0)};
  int nf = 0;
  for (int m = 0; m < M; ++m) {
#pragma unroll
    for (int k = 0; k < 3; ++k) tan.dy[k] = mk(0.0);
    int nfe = 0;
    rk45_generic<3, TPB>(A, dtaus[m], f, K, &nfe, &tan);
    nf += nfe;
    dlog_mgf_theta[(size_t)m * P + p] = (tan.dy[0] + tan.dy[1] * c.lambda_p) + tan.dy[2] * c.lambda_m;
  }
  if (nfev) nfev[p] = nf;
}

// The Heston closed form on dual numbers in tau: (a, b) carried over the earlier slices with their derivatives zeroed at every slice
// start, then the slice's step with d tau = 1.  dlog_mgf_theta [M][P] = da + db v0.
__global__ void heston_mgf_theta_kernel(const cd* __restrict__ phi, int P, int M, const double* __restrict__ dtaus, b200sv_heston_params hp,
                                        cd* __restrict__ dlog_mgf_theta) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const HestonClosedForm<dcd, dcd> cf(dmk(mk(hp.theta)), dmk(mk(hp.kappa)), dmk(mk(hp.rho)), dmk(mk(hp.volvol)), phi[p], mk(0.0));
  dcd a = dmk(mk(0.0)), b = dmk(mk(0.0));
  for (int mm = 0; mm < M; ++mm) {
    a.d = mk(0.0);
    b.d = mk(0.0);
    cf.step(dmk(mk(dtaus[mm]), mk(1.0)), a, b);
    dlog_mgf_theta[(size_t)mm * P + p] = a.d + b.d * hp.v0;
  }
}

// --------------------------------------------------------------------------------------------------------------------
// host side
// --------------------------------------------------------------------------------------------------------------------
// Latency regime (few grid points in total): lane-parallel kernel; throughput regime (batches, the 40000-point psi grid): one thread per
// point.  B200SV_MGF_LANES=0/1 overrides the choice (A/B timing in tools/bench_mgf.py).
static bool use_lane_kernel(long long points) {
  static const int forced = [] {
    const char* e = getenv("B200SV_MGF_LANES");
    return e ? atoi(e) : -1;
  }();
  if (forced >= 0) return forced != 0;
  return points <= 8192;
}

// dense M / L / H of affine_expansion.py:139-184 from the row tables (parity entry b200sv_logsv_ode_terms)
template <int N>
__global__ void logsv_ode_terms_kernel(const cd* __restrict__ phi, const cd* __restrict__ psi, int P, LogsvModel m, cd* __restrict__ M_out,
                                       cd* __restrict__ L_out, cd* __restrict__ H_out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const cd ph = phi[p], ps = psi ? psi[p] : mk(0.0);
  cd* Mo = M_out + (size_t)p * N * N * N;
  cd* Lo = L_out + (size_t)p * N * N;
  for (int i = 0; i < N * N * N; ++i) Mo[i] = mk(0.0);
  for (int i = 0; i < N * N; ++i) Lo[i] = mk(0.0);
  for (int k = 0; k < N; ++k) {
    const LaneRow<N> r = make_lane_row<N>(k, m, ph, ps);
    for (int t = 0; t < r.nq; ++t) {
      const int i = r.qi[t], j = r.qj[t];
      if (i == j) {
        Mo[(k * N + i) * N + i] = mk(r.q[t]);
      } else {          // the row tables carry off-diagonal pairs doubled: A_i A_j (M_ij + M_ji)
        Mo[(k * N + i) * N + j] = mk(0.5 * r.q[t]);
        Mo[(k * N + j) * N + i] = mk(0.5 * r.q[t]);
      }
    }
    for (int t = 0; t < r.nl; ++t) Lo[k * N + r.li[t]] = r.l[t];
    H_out[(size_t)p * N + k] = r.h;
  }
}

// func_rhs (affine_expansion.py:187-205) through the production right-hand side
template <int N>
__global__ void logsv_ode_rhs_kernel(const cd* __restrict__ phi, const cd* __restrict__ psi, int P, LogsvModel m, const cd* __restrict__ A_in,
                                     cd* __restrict__ rhs_out) {
  __shared__ cd coef_smem[14 * 64];
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  store_coef<64>(coef_smem + threadIdx.x, make_coef(m, phi[p], psi ? psi[p] : mk(0.0)));
  const CoefView<64> c{coef_smem + threadIdx.x};
  cd A[N], out[N];
#pragma unroll
  for (int k = 0; k < N; ++k) A[k] = A_in[(size_t)p * N + k];
  rhs<N, 64>(A, m, c, out);
#pragma unroll
  for (int k = 0; k < N; ++k) rhs_out[(size_t)p * N + k] = out[k];
}

// func_rhs with caller-supplied dense tensors (the reference signature): rhs[p][k] = A_p^T M[k] A_p + (L A_p)[k] + H[k]
__global__ void ode_rhs_dense_kernel(const cd* __restrict__ A, int P, int n, const cd* __restrict__ M, const cd* __restrict__ L,
                                     const cd* __restrict__ H, cd* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P * n) return;
  const int p = idx / n, k = idx % n;
  const cd* a = A + (size_t)p * n;
  cd acc = mk(0.0);
  for (int i = 0; i < n; ++i) {          // A^T M[k] A: row-by-row, as numpy's A0.T @ M[n_] @ A0 contracts (vector-matrix, then dot)
    cd row = mk(0.0);
    for (int j = 0; j < n; ++j) row = row + a[j] * M[((size_t)k * n + j) * n + i];
    acc = acc + row * a[i];
  }
  cd lin = mk(0.0);
  for (int j = 0; j < n; ++j) lin = lin + L[(size_t)k * n + j] * a[j];
  out[idx] = (acc + lin) + H[k];
}

// --------------------------------------------------------------------------------------------------------------------
// semi-analytic branch: solve_analytic_ode_for_a (pricers/logsv/affine_expansion.py:306-384), is_analytic=True
// --------------------------------------------------------------------------------------------------------------------
// The reference steps A' = A^T M A + L A + H on a business-day grid (nb_steps = ceil(260 dtau)): the linear part exactly -- through
// eig(L), v diag(exp(w dt)) v^-1 and v diag((exp(w dt) - 1)/w) v^-1 with the zero eigenvalue's entry set to 0 -- and the quadratic part by
// 10 unchecked fixed-point sweeps per step, quadratic term times plain dt; row 0 of the right-hand side is (H_0 + quad_0) dt.
// Here the two matrices are formed WITHOUT an eigendecomposition: v diag(e^{w dt}) v^-1 = expm(L dt) =: E, and because column 0 of L is zero
// (nothing depends on A_0) the null eigenvector is e_0, so rows 1.. of the second matrix equal rows 1.. of Psi = int_0^dt e^{L s} ds
// (the projector that the reference removes has only row 0, and row 0 is overwritten anyway).  E and Psi come from a degree-18 Taylor series
// of the scaled matrix and s doublings  Psi_{2h} = (I + E_h) Psi_h,  E_{2h} = E_h^2  -- 5x5 complex products in thread-local memory, once per
// (grid point, maturity).  Agreement with the reference's LAPACK route is limited by the conditioning of ITS eigenvector matrix (1e-10 on
// the goldens).  vol_backbone_eta is ignored on this branch as in the reference (:340-348: not passed to func_a_ode_quadratic_terms).
template <int N>
__device__ void cmat_mul(const cd (&A)[N][N], const cd (&B)[N][N], cd (&C)[N][N]) {
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) {
      cd acc = mk(0.0);
      for (int k = 0; k < N; ++k) acc = acc + A[i][k] * B[k][j];
      C[i][j] = acc;
    }
}

template <int N>
__global__ void __launch_bounds__(64) logsv_mgf_analytic_kernel(const cd* __restrict__ phi, const cd* __restrict__ psi, int P, LogsvModel m, double dtau,
                                                                int year_days, const cd* __restrict__ a_in, cd* __restrict__ a_out,
                                                                cd* __restrict__ log_mgf, double y) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const cd ph = phi[p], ps = psi ? psi[p] : mk(0.0);
  const int nb_steps = (int)ceil((double)year_days * dtau);
  const double dt = dtau / (double)nb_steps;
  // rows of the system (the same tables the RK45 kernels integrate) -> dense L, H
  LaneRow<N> rows[N];
  cd L[N][N], H[N];
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) L[i][j] = mk(0.0);
  double nrm = 0.0;
  for (int k = 0; k < N; ++k) {
    rows[k] = make_lane_row<N>(k, m, ph, ps);
    for (int t = 0; t < rows[k].nl; ++t) L[k][rows[k].li[t]] = rows[k].l[t];
    H[k] = rows[k].h;
    double rs = 0.0;
    for (int j = 0; j < N; ++j) rs += cabs_(L[k][j]);
    nrm = fmax(nrm, rs);
  }
  // scaling: ||L h||_inf <= 1/2
  int sq = 0;
  double h = dt;
  while (nrm * h > 0.5 && sq < 40) {
    h *= 0.5;
    ++sq;
  }
  cd X[N][N], E[N][N], Psi[N][N], T1[N][N], T2[N][N];
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) {
      X[i][j] = h * L[i][j];
      E[i][j] = mk(i == j ? 1.0 : 0.0);
      Psi[i][j] = mk(i == j ? h : 0.0);
      T1[i][j] = E[i][j];                     // running term X^k / k!
    }
  for (int k = 1; k <= 18; ++k) {             // E = sum X^k/k!,  Psi = h sum X^k/(k+1)!
    cmat_mul<N>(T1, X, T2);
    for (int i = 0; i < N; ++i)
      for (int j = 0; j < N; ++j) {
        T1[i][j] = (1.0 / k) * T2[i][j];
        E[i][j] = E[i][j] + T1[i][j];
        Psi[i][j] = Psi[i][j] + (h / (k + 1)) * T1[i][j];
      }
  }
  for (int d = 0; d < sq; ++d) {              // doubling
    for (int i = 0; i < N; ++i)
      for (int j = 0; j < N; ++j) T1[i][j] = E[i][j] + mk(i == j ? 1.0 : 0.0);
    cmat_mul<N>(T1, Psi, T2);
    cmat_mul<N>(E, E, T1);
    for (int i = 0; i < N; ++i)
      for (int j = 0; j < N; ++j) {
        Psi[i][j] = T2[i][j];
        E[i][j] = T1[i][j];
      }
  }
  cd g[N];                                    // rows 1.. of (m_rhs @ H)
  for (int k = 0; k < N; ++k) {
    cd acc = mk(0.0);
    for (int j = 0; j < N; ++j) acc = acc + Psi[k][j] * H[j];
    g[k] = acc;
  }
  cd a[N], fp[N], q[N];
  for (int k = 0; k < N; ++k) a[k] = a_in[(size_t)p * N + k];
  for (int t = 0; t < nb_steps; ++t) {
    for (int k = 0; k < N; ++k) fp[k] = a[k];
    cd Ea[N];
    for (int k = 0; k < N; ++k) {
      cd acc = mk(0.0);
      for (int j = 0; j < N; ++j) acc = acc + E[k][j] * a[j];
      Ea[k] = acc;
    }
    for (int it = 0; it < 10; ++it) {         // nfp = 10, no convergence test (:365)
      for (int k = 0; k < N; ++k) {
        cd acc = mk(0.0);
        for (int u = 0; u < rows[k].nq; ++u) acc = acc + rows[k].q[u] * (fp[rows[k].qi[u]] * fp[rows[k].qj[u]]);
        q[k] = acc;
      }
      fp[0] = Ea[0] + dt * (H[0] + q[0]);
      for (int k = 1; k < N; ++k) fp[k] = Ea[k] + (g[k] + dt * q[k]);
    }
    for (int k = 0; k < N; ++k) a[k] = fp[k];
  }
  double yk = 1.0;
  cd lm = mk(0.0);
  for (int k = 0; k < N; ++k) {
    a_out[(size_t)p * N + k] = a[k];
    lm = lm + yk * a[k];
    yk *= y;
  }
  log_mgf[p] = lm;
}

// --------------------------------------------------------------------------------------------------------------------
// stiff branch: solve_ivp(method="BDF", jac=func_rhs_jac) as used by solve_ode_for_a(is_stiff_solver=True) (affine_expansion.py:229-303)
// --------------------------------------------------------------------------------------------------------------------
// A clone of the CONTROL LAW of scipy.integrate.BDF (scipy 1.18.1, scipy/integrate/_ivp/bdf.py:14-60, 186-230, 317-455; select_initial_step
// with order 1, common.py:68-134; rtol 1e-3 / atol 1e-6): variable order 1..5 NDF with quasi-constant step size, the differences array D and
// its rescaling matrices (change_D), simplified Newton with at most 4 iterations on an LU of I - c J that is KEPT across steps and across
// error rejections (bdf.py resets it only when the step size changes for other reasons), Jacobian refreshed only after a failed Newton
// solve, order selection from the three error norms after order + 1 equal steps.  Parity with the reference means reproducing its accepted
// steps, so every branch of the step routine is mirrored; floating-point differences (LAPACK's blocked zgetrf / BLAS dot products vs the
// scalar loops here) stay at the 1e-15 level because the decisions are thresholds on norms (tests: 1e-10 against the reference goldens).
// One thread = one grid point; D (8 x N complex), J and LU live in thread-local memory -- this is the reference's non-default branch, 1000
// independent stiff solves of ~30 steps each, not a throughput path.
template <int N>
struct BdfState {
  cd D[8][N];
  cd J[N][N], LU[N][N];
  int piv[N];
  bool lu_valid;
};

__device__ __forceinline__ double cabs1(cd a) { return fabs(a.re) + fabs(a.im); }     // LAPACK izamax's magnitude

template <int N>
__device__ void bdf_lu_factor(BdfState<N>& s, double c) {             // LU of I - c J, partial pivoting (zgetrf semantics)
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) s.LU[i][j] = mk(i == j ? 1.0 : 0.0) - c * s.J[i][j];
  for (int k = 0; k < N; ++k) {
    int p = k;
    double best = cabs1(s.LU[k][k]);
    for (int i = k + 1; i < N; ++i) {
      const double v = cabs1(s.LU[i][k]);
      if (v > best) {
        best = v;
        p = i;
      }
    }
    s.piv[k] = p;
    if (p != k)
      for (int j = 0; j < N; ++j) {
        const cd t = s.LU[k][j];
        s.LU[k][j] = s.LU[p][j];
        s.LU[p][j] = t;
      }
    const cd inv = mk(1.0) / s.LU[k][k];
    for (int i = k + 1; i < N; ++i) {
      s.LU[i][k] = s.LU[i][k] * inv;
      for (int j = k + 1; j < N; ++j) s.LU[i][j] = s.LU[i][j] - s.LU[i][k] * s.LU[k][j];
    }
  }
  s.lu_valid = true;
}

template <int N>
__device__ void bdf_lu_solve(const BdfState<N>& s, cd (&b)[N]) {
  for (int k = 0; k < N; ++k) {
    const int p = s.piv[k];
    if (p != k) {
      const cd t = b[k];
      b[k] = b[p];
      b[p] = t;
    }
  }
  for (int i = 1; i < N; ++i)
    for (int j = 0; j < i; ++j) b[i] = b[i] - s.LU[i][j] * b[j];
  for (int i = N - 1; i >= 0; --i) {
    for (int j = i + 1; j < N; ++j) b[i] = b[i] - s.LU[i][j] * b[j];
    b[i] = b[i] / s.LU[i][i];
  }
}

// func_rhs_jac (affine_expansion.py:208-225): J = 2 M[k] A + L, from the row tables
template <int N>
__device__ void bdf_jacobian(BdfState<N>& s, const cd (&A)[N], const LogsvModel& m, cd phi, cd psi) {
  for (int k = 0; k < N; ++k) {
    for (int j = 0; j < N; ++j) s.J[k][j] = mk(0.0);
    const LaneRow<N> r = make_lane_row<N>(k, m, phi, psi);
    for (int t = 0; t < r.nq; ++t) {
      const int i = r.qi[t], j = r.qj[t];
      if (i == j) {
        s.J[k][i] = s.J[k][i] + (2.0 * r.q[t]) * A[i];
      } else {                       // the tables carry off-diagonal pairs doubled: q A_i A_j with q = M_ij + M_ji
        s.J[k][i] = s.J[k][i] + r.q[t] * A[j];
        s.J[k][j] = s.J[k][j] + r.q[t] * A[i];
      }
    }
    for (int t = 0; t < r.nl; ++t) s.J[k][r.li[t]] = s.J[k][r.li[t]] + r.l[t];
  }
}

// change_D (bdf.py:28-33): D[:order+1] <- (R U)^T D[:order+1],  R = compute_R(order, factor), U = compute_R(order, 1)
template <int N>
__device__ void bdf_change_D(BdfState<N>& s, int order, double factor) {
  double R[6][6], U[6][6], RU[6][6];
  for (int j = 0; j <= order; ++j) {
    R[0][j] = 1.0;
    U[0][j] = 1.0;
  }
  for (int i = 1; i <= order; ++i) {
    R[i][0] = 0.0;                  // M[i][0] = 0 => cumprod is 0 from row 1 on
    U[i][0] = 0.0;
    for (int j = 1; j <= order; ++j) {
      R[i][j] = R[i - 1][j] * (((double)(i - 1) - factor * (double)j) / (double)i);
      U[i][j] = U[i - 1][j] * (((double)(i - 1) - (double)j) / (double)i);
    }
  }
  for (int i = 0; i <= order; ++i)
    for (int j = 0; j <= order; ++j) {
      double acc = 0.0;
      for (int k = 0; k <= order; ++k) acc += R[i][k] * U[k][j];
      RU[i][j] = acc;
    }
  cd Dn[6][N];
  for (int i = 0; i <= order; ++i)
    for (int c = 0; c < N; ++c) {
      cd acc = mk(0.0);
      for (int k = 0; k <= order; ++k) acc = acc + RU[k][i] * s.D[k][c];
      Dn[i][c] = acc;
    }
  for (int i = 0; i <= order; ++i)
    for (int c = 0; c < N; ++c) s.D[i][c] = Dn[i][c];
}

template <int N>
__device__ double bdf_norm_scaled(const cd (&v)[N], const double (&scale)[N]) {       // norm(v / scale) = ||.||_2 / sqrt(n)
  double acc = 0.0;
  for (int k = 0; k < N; ++k) {
    const double re = v[k].re / scale[k], im = v[k].im / scale[k];
    acc += re * re + im * im;
  }
  return sqrt(acc) / sqrt((double)N);
}

// returns 0 ok, 1 step size underflow (TOO_SMALL_STEP: the reference keeps the last accepted state)
template <int N, int TPB>
__device__ int bdf_integrate(cd (&y)[N], double T, const LogsvModel& m, const CoefView<TPB>& c, cd phi, cd psi, BdfState<N>& s) {
  const double gamma[6] = {0.0, 1.0, 1.5, 1.5 + 1.0 / 3.0, 1.5 + 1.0 / 3.0 + 0.25, 1.5 + 1.0 / 3.0 + 0.25 + 0.2};
  const double kappa[6] = {0.0, -0.1850, -1.0 / 9.0, -0.0823, -0.0415, 0.0};
  double alpha[6], error_const[7];
  for (int i = 0; i < 6; ++i) {
    alpha[i] = (1.0 - kappa[i]) * gamma[i];
    error_const[i] = kappa[i] * gamma[i] + 1.0 / (double)(i + 1);
  }
  const double newton_tol = 0.03;       // max(10 EPS / rtol, min(0.03, sqrt(rtol)))
  cd f[N];
  rhs<N, TPB>(y, m, c, f);
  double h_abs;
  {  // select_initial_step(order = 1)
    double scale[N];
    for (int k = 0; k < N; ++k) scale[k] = kAtol + cmod(y[k]) * kRtol;
    const double d0 = bdf_norm_scaled<N>(y, scale), d1 = bdf_norm_scaled<N>(f, scale);
    double h0 = (d0 < 1e-5 || d1 < 1e-5) ? 1e-6 : 0.01 * d0 / d1;
    h0 = fmin(h0, T);
    cd y1[N], f1[N];
    for (int k = 0; k < N; ++k) y1[k] = y[k] + h0 * f[k];
    rhs<N, TPB>(y1, m, c, f1);
    for (int k = 0; k < N; ++k) f1[k] = f1[k] - f[k];
    const double d2 = bdf_norm_scaled<N>(f1, scale) / h0;
    const double h1 = (d1 <= 1e-15 && d2 <= 1e-15) ? fmax(1e-6, h0 * 1e-3) : sqrt(0.01 / fmax(d1, d2));
    h_abs = fmin(fmin(100.0 * h0, h1), T);
  }
  bdf_jacobian<N>(s, y, m, phi, psi);
  for (int i = 0; i < 8; ++i)
    for (int k = 0; k < N; ++k) s.D[i][k] = mk(0.0);
  for (int k = 0; k < N; ++k) {
    s.D[0][k] = y[k];
    s.D[1][k] = h_abs * f[k];
  }
  int order = 1, n_equal_steps = 0;
  s.lu_valid = false;
  double t = 0.0;
  for (int guard = 0; t < T && guard < 100000; ++guard) {
    // ---- _step_impl (bdf.py:317-455)
    const double min_step = 10.0 * (__longlong_as_double(__double_as_longlong(t) + 1) - t);
    if (h_abs < min_step) {
      bdf_change_D<N>(s, order, min_step / h_abs);
      h_abs = min_step;
      n_equal_steps = 0;
    }
    bool current_jac = false;
    bool accepted = false;
    double t_new = t, safety = 0.0, error_norm = 0.0;
    double scale[N];
    cd y_new[N], d[N];
    while (!accepted) {
      if (h_abs < min_step) return 1;
      t_new = t + h_abs;
      if (t_new - T > 0.0) {
        t_new = T;
        bdf_change_D<N>(s, order, fabs(t_new - t) / h_abs);
        n_equal_steps = 0;
        s.lu_valid = false;
      }
      const double h = t_new - t;
      h_abs = fabs(h);
      cd y_predict[N], psi_v[N];
      for (int k = 0; k < N; ++k) {
        cd acc = s.D[0][k];
        for (int i = 1; i <= order; ++i) acc = acc + s.D[i][k];
        y_predict[k] = acc;
        scale[k] = kAtol + kRtol * cmod(acc);
        cd ps = mk(0.0);
        for (int i = 1; i <= order; ++i) ps = ps + gamma[i] * s.D[i][k];
        psi_v[k] = mk(ps.re / alpha[order], ps.im / alpha[order]);      // numpy divides (dot(...) / alpha[order]): no reciprocal multiply
      }
      const double cc = h / alpha[order];
      bool converged = false;
      int n_iter = 0;
      while (!converged) {
        if (!s.lu_valid) bdf_lu_factor<N>(s, cc);
        // ---- solve_bdf_system (bdf.py:36-72)
        for (int k = 0; k < N; ++k) {
          d[k] = mk(0.0);
          y_new[k] = y_predict[k];
        }
        double dy_norm_old = -1.0;
        for (int k_it = 0; k_it < 4; ++k_it) {
          cd fn[N];
          rhs<N, TPB>(y_new, m, c, fn);
          bool finite = true;
          for (int k = 0; k < N; ++k) finite = finite && isfinite(fn[k].re) && isfinite(fn[k].im);
          if (!finite) break;
          cd dy[N];
          for (int k = 0; k < N; ++k) dy[k] = (cc * fn[k] - psi_v[k]) - d[k];
          bdf_lu_solve<N>(s, dy);
          const double dy_norm = bdf_norm_scaled<N>(dy, scale);
          const bool have_rate = dy_norm_old >= 0.0;
          const double rate = have_rate ? dy_norm / dy_norm_old : 0.0;
          if (have_rate && (rate >= 1.0 || pow(rate, (double)(4 - k_it)) / (1.0 - rate) * dy_norm > newton_tol)) break;
          for (int k = 0; k < N; ++k) {
            y_new[k] = y_new[k] + dy[k];
            d[k] = d[k] + dy[k];
          }
          n_iter = k_it + 1;
          if (dy_norm == 0.0 || (have_rate && rate / (1.0 - rate) * dy_norm < newton_tol)) {
            converged = true;
            break;
          }
          dy_norm_old = dy_norm;
        }
        if (!converged) {
          if (current_jac) break;
          bdf_jacobian<N>(s, y_predict, m, phi, psi);
          s.lu_valid = false;
          current_jac = true;
        }
      }
      if (!converged) {
        h_abs *= 0.5;
        bdf_change_D<N>(s, order, 0.5);
        n_equal_steps = 0;
        s.lu_valid = false;
        continue;
      }
      safety = 0.9 * (2.0 * 4.0 + 1.0) / (2.0 * 4.0 + (double)n_iter);
      for (int k = 0; k < N; ++k) scale[k] = kAtol + kRtol * cmod(y_new[k]);
      cd err[N];
      for (int k = 0; k < N; ++k) err[k] = error_const[order] * d[k];
      error_norm = bdf_norm_scaled<N>(err, scale);
      if (error_norm > 1.0) {
        const double factor = fmax(0.2, safety * pow(error_norm, -1.0 / (double)(order + 1)));
        h_abs *= factor;
        bdf_change_D<N>(s, order, factor);
        n_equal_steps = 0;            // LU is deliberately NOT invalidated here (bdf.py:398-403)
      } else {
        accepted = true;
      }
    }
    ++n_equal_steps;
    t = t_new;
    for (int k = 0; k < N; ++k) {
      y[k] = y_new[k];
      s.D[order + 2][k] = d[k] - s.D[order + 1][k];
      s.D[order + 1][k] = d[k];
    }
    for (int i = order; i >= 0; --i)
      for (int k = 0; k < N; ++k) s.D[i][k] = s.D[i][k] + s.D[i + 1][k];
    if (n_equal_steps < order + 1) continue;
    double en[3];
    {
      cd e[N];
      if (order > 1) {
        for (int k = 0; k < N; ++k) e[k] = error_const[order - 1] * s.D[order][k];
        en[0] = bdf_norm_scaled<N>(e, scale);
      } else {
        en[0] = INFINITY;
      }
      en[1] = error_norm;
      if (order < 5) {
        for (int k = 0; k < N; ++k) e[k] = error_const[order + 1] * s.D[order + 2][k];
        en[2] = bdf_norm_scaled<N>(e, scale);
      } else {
        en[2] = INFINITY;
      }
    }
    double factors[3], best = -1.0;
    int arg = 0;
    for (int i = 0; i < 3; ++i) {
      factors[i] = pow(en[i], -1.0 / (double)(order + i));     // 0 -> inf, inf -> 0 (numpy with divide='ignore')
      if (factors[i] > best) {                                   // np.argmax: first maximum
        best = factors[i];
        arg = i;
      }
    }
    order += arg - 1;
    const double factor = fmin(10.0, safety * best);
    h_abs *= factor;
    bdf_change_D<N>(s, order, factor);
    n_equal_steps = 0;
    s.lu_valid = false;
  }
  return 0;
}

template <int N>
__global__ void __launch_bounds__(64) logsv_mgf_bdf_kernel(const cd* __restrict__ phi, const cd* __restrict__ psi, int P, LogsvModel m, double dtau,
                                                           const cd* __restrict__ a_in, cd* __restrict__ a_out, cd* __restrict__ log_mgf, double y,
                                                           int* __restrict__ status) {
  __shared__ cd coef_smem[14 * 64];
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const cd ph = phi[p], ps = psi ? psi[p] : mk(0.0);
  store_coef<64>(coef_smem + threadIdx.x, make_coef(m, ph, ps));
  const CoefView<64> c{coef_smem + threadIdx.x};
  cd A[N];
  for (int k = 0; k < N; ++k) A[k] = a_in[(size_t)p * N + k];
  BdfState<N> st;
  const int rc = bdf_integrate<N, 64>(A, dtau, m, c, ph, ps, st);
  if (status) status[p] = rc;
  double yk = 1.0;
  cd lm = mk(0.0);
  for (int k = 0; k < N; ++k) {
    a_out[(size_t)p * N + k] = A[k];
    lm = lm + yk * A[k];
    yk *= y;
  }
  log_mgf[p] = lm;
}

static int mgf_block_threads(int P) {
  const int sms = device_sm_count();
  int t = 4;
  while (t < 64 && t * sms < P) t <<= 1;
  return t;
}

// np.linspace(0, stop, P): y[i] = i*step, step = stop/(P-1), last = stop; phi = re + 1j*p (utils/mgf_pricer.py:22-33)
static void build_phi(double vol_scaler, bool spot, int P, std::vector<double>& phi) {
  phi.resize(2 * (size_t)P);
  const double stop = 5.6 / vol_scaler, step = stop / (double)(P - 1);
  for (int i = 0; i < P; ++i) {
    phi[2 * i] = spot ? -0.5 : 0.5;
    phi[2 * i + 1] = (double)i * step;
  }
  phi[2 * (size_t)(P - 1) + 1] = stop;
}

// re + 1j*linspace(0, stop, P)  (get_psi_grid: -0.5 + 1j*linspace(0, 4000, 40000), utils/mgf_pricer.py:37-47)
static void build_grid(double re, double stop, int P, std::vector<double>& g) {
  g.resize(2 * (size_t)P);
  const double step = stop / (double)(P - 1);
  for (int i = 0; i < P; ++i) {
    g[2 * i] = re;
    g[2 * i + 1] = (double)i * step;
  }
  g[2 * (size_t)(P - 1) + 1] = stop;
}

static int check_qvar_types(const int8_t* types, int n) {
  for (int j = 0; j < n; ++j)
    if (types[j] != B200SV_CALL) return fail(-5, "not implemented");      // utils/mgf_pricer.py:349-358: only 'C'
  return 0;
}

static int check_fourier_types(const int8_t* types, int n, bool spot) {
  for (int j = 0; j < n; ++j) {
    if (types[j] < 0 || types[j] > 3) return fail(-5, "not implemented");
    // MMA measure rejects inverse payoffs (utils/mgf_pricer.py:206-212); the inverse measure accepts C == IC, P == IP (:214-217)
    if (spot && types[j] >= 2) return fail(-5, "not implemented");
  }
  return 0;
}

// the gamma slice pricer prices 'C' / 'P' under the spot measure only (utils/mgf_pricer.py:310-318)
static int check_gamma_types(const int8_t* types, int n, bool spot) {
  if (!spot) return fail(-5, "not implemented");
  for (int j = 0; j < n; ++j)
    if (types[j] != B200SV_CALL && types[j] != B200SV_PUT) return fail(-5, "not implemented");
  return 0;
}

static bool all_half_re(const double* phi, int P) {
  for (int i = 0; i < P; ++i)
    if (std::fabs(phi[2 * i]) != 0.5) return false;
  return true;
}

// caller arrays of complex numbers are interleaved doubles
static const cd* cplx(const double* p) { return reinterpret_cast<const cd*>(p); }
static cd* cplx(double* p) { return reinterpret_cast<cd*>(p); }

// ---- kernel maps: one instantiation per expansion order N (3 or 5) and block size (mgf_block_threads: 4 .. 64) ----
using LogsvMgfKernel = decltype(&logsv_mgf_kernel<5, 64>);
static LogsvMgfKernel logsv_mgf_kernel_for(int N, int tpb) {
  switch (tpb) {
    case 4: return N == 5 ? logsv_mgf_kernel<5, 4> : logsv_mgf_kernel<3, 4>;
    case 8: return N == 5 ? logsv_mgf_kernel<5, 8> : logsv_mgf_kernel<3, 8>;
    case 16: return N == 5 ? logsv_mgf_kernel<5, 16> : logsv_mgf_kernel<3, 16>;
    case 32: return N == 5 ? logsv_mgf_kernel<5, 32> : logsv_mgf_kernel<3, 32>;
    default: return N == 5 ? logsv_mgf_kernel<5, 64> : logsv_mgf_kernel<3, 64>;
  }
}

using HawkesMgfKernel = decltype(&hawkes_mgf_kernel<64>);
static HawkesMgfKernel hawkes_mgf_kernel_for(int tpb) {
  switch (tpb) {
    case 4: return hawkes_mgf_kernel<4>;
    case 8: return hawkes_mgf_kernel<8>;
    case 16: return hawkes_mgf_kernel<16>;
    case 32: return hawkes_mgf_kernel<32>;
    default: return hawkes_mgf_kernel<64>;
  }
}

// logsv_mgf_kernel (or its lane-parallel form) over B parameter sets; block size from the B * P points in flight
static void launch_logsv_mgf(int N, cudaStream_t st, const cd* phi, const cd* psi, int P, int M, const ChainSpec* spec, const cd* a_in,
                             cd* a_out, cd* lm, double y, int B = 1, const double* yb = nullptr, int phi_stride = 0) {
  if (use_lane_kernel((long long)P * B)) {
    const int per_block = 32 / (N == 5 ? 8 : 4) * kLaneWarpsPerBlock;      // grid points per warp x warps
    const auto lanes = N == 5 ? logsv_mgf_lanes_kernel<5> : logsv_mgf_lanes_kernel<3>;
    lanes<<<dim3((P + per_block - 1) / per_block, B), 32 * kLaneWarpsPerBlock, 0, st>>>(phi, psi, P, M, spec, a_in, a_out, lm, y, nullptr, yb,
                                                                                        phi_stride);
    return;
  }
  static const bool set_major = [] {
    const char* e = getenv("B200SV_MGF_SET_MAJOR");      // A/B timing switch (tools/bench_calibration.py); default on
    return !e || atoi(e) != 0;
  }();
  const int tpb = mgf_block_threads((int)std::min<long long>((long long)B * P, 1 << 30));
  const int smB = (B > 1 && set_major) ? B : 0;
  const dim3 grid = smB ? dim3((unsigned)(((long long)B * P + tpb - 1) / tpb), 1) : dim3((P + tpb - 1) / tpb, B);
  const LogsvMgfKernel k = logsv_mgf_kernel_for(N, tpb);
  k<<<grid, tpb, 0, st>>>(phi, psi, P, M, spec, a_in, a_out, lm, y, nullptr, nullptr, yb, phi_stride, smB);
}

static void launch_hawkes_mgf(cudaStream_t st, const cd* phi, const cd* psi, int P, int M, const double* dtaus, const HawkesMgfConsts& c,
                              const cd* a_in, cd* a_out, cd* lm, int restart) {
  const int tpb = mgf_block_threads(P);
  const HawkesMgfKernel k = hawkes_mgf_kernel_for(tpb);
  k<<<(P + tpb - 1) / tpb, tpb, 0, st>>>(phi, psi, P, M, dtaus, c, a_in, a_out, lm, restart, nullptr);
}

// hawkes_mgf_sets_kernel over the B * P (set, point) threads of B sets; block size as for hawkes_mgf_kernel, from the threads in flight.
// RESTART: set_m0 [B + 1] (device) places each set's rows, see the kernel.
template <bool RESTART = false>
static void launch_hawkes_mgf_sets(cudaStream_t st, const cd* phi, int P, int M, const double* dtaus, const HawkesMgfConsts* consts, int B,
                                   int phi_stride, cd* lm, const int* set_m0 = nullptr) {
  const long long n = (long long)B * P;
  const int tpb = mgf_block_threads((int)std::min<long long>(n, 1 << 30));
  decltype(&hawkes_mgf_sets_kernel<64, RESTART>) k;
  switch (tpb) {
    case 4: k = hawkes_mgf_sets_kernel<4, RESTART>; break;
    case 8: k = hawkes_mgf_sets_kernel<8, RESTART>; break;
    case 16: k = hawkes_mgf_sets_kernel<16, RESTART>; break;
    case 32: k = hawkes_mgf_sets_kernel<32, RESTART>; break;
    default: k = hawkes_mgf_sets_kernel<64, RESTART>;
  }
  k<<<(unsigned)((n + tpb - 1) / tpb), tpb, 0, st>>>(phi, P, M, dtaus, consts, B, phi_stride, lm, set_m0);
}

// hawkes_mgf_tangent_kernel<TPB, Phi> over the P * (13 + Phi) (point, direction) threads; block size as for hawkes_mgf_kernel, from the
// threads in flight
template <bool Phi>
static void launch_hawkes_mgf_tangent(cudaStream_t st, const cd* phi, int P, int M, const double* dtaus, const HawkesMgfConsts& c,
                                      const HawkesTangentDirs& dirs, int restart, cd* dlm, cd* lm, int* nfev) {
  const int n = P * (kHawkesOdeDirs + Phi), tpb = mgf_block_threads(n);
  decltype(&hawkes_mgf_tangent_kernel<64, Phi>) k;
  switch (tpb) {
    case 4: k = hawkes_mgf_tangent_kernel<4, Phi>; break;
    case 8: k = hawkes_mgf_tangent_kernel<8, Phi>; break;
    case 16: k = hawkes_mgf_tangent_kernel<16, Phi>; break;
    case 32: k = hawkes_mgf_tangent_kernel<32, Phi>; break;
    default: k = hawkes_mgf_tangent_kernel<64, Phi>;
  }
  k<<<(n + tpb - 1) / tpb, tpb, 0, st>>>(phi, P, M, dtaus, c, dirs, restart, dlm, lm, nullptr, nfev);
}

// ---- chain preparation ----
// Default transform-grid scale when the caller passes vol_scaler <= 0; t0 is the first (shortest) maturity.
static double default_vol_scaler(const b200sv_logsv_params& p, double t0) {      // logsv_pricer.py:664-666
  return p.sigma0 * std::sqrt(std::min(t0, 0.5 / 12.0));
}
static double default_vol_scaler(const b200sv_heston_params& p, double t0) {     // heston_pricer.py:234-235
  return std::min(0.3, std::sqrt(p.v0 * t0));
}
static double default_vol_scaler(const b200sv_hawkes_params& p, double t0) {     // hawkes_jd_pricer.py:360-362
  return std::min(std::max(p.sigma, 0.2), 0.5) * std::sqrt(std::min(t0, 1.0 / 12.0));
}

enum class ChainTypes { kFourier, kQvar, kGamma };   // which payoffs the route prices: check_fourier_types / _qvar_ / _gamma_

// One option chain of a Fourier chain pricer, validated once, with everything its launches read: the maturity increments, the transform
// grid(s) and one strike row per (parameter set, strike).  init() checks the sizes; build() the option types, maturities and strikes.
struct FourierChain {
  bool batch = false, spot = true, qvar = false, per_set_grid = false;
  int B = 1, M = 0, P = 0, Jtot = 0;
  std::vector<double> dtaus, phi, psi;    // phi [G][P] complex (G = B with a per-set grid, else 1); psi [P] under Q_VAR only
  std::vector<StrikeSpec> ss;             // [B][Jtot]: slice b * M + m, grid b (per-set grid) or 0
  std::vector<SumSpec> qs;                // [Jtot], Q_VAR only

  // batch: the B sets of b200sv_*_price_chain_batch, which also need at least one strike
  int init(bool is_batch, int nsets, int nmat, int npoints, const int* offsets) {
    batch = is_batch;
    B = nsets;
    M = nmat;
    P = npoints;
    if (batch)
      B200SV_REQUIRE(B >= 1 && B <= 65535 && M >= 1 && P >= 3, "1 <= B <= 65535, M >= 1, P >= 3");
    else
      B200SV_REQUIRE(M >= 1 && P >= 3, "M >= 1, P >= 3");
    Jtot = offsets[M] - offsets[0];
    if (batch) B200SV_REQUIRE(Jtot >= 1, "the chain has no strikes");
    return 0;
  }

  template <class Params>
  int build(const Params* params, const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
            const double* strikes, const int8_t* types, bool is_spot, ChainTypes payoffs, double vol_scaler) {
    spot = is_spot;
    qvar = payoffs == ChainTypes::kQvar;
    B200SV_REQUIRE(Jtot == 0 || types, "null pointer");
    const int8_t* t = types + offsets[0];
    if (int rc = qvar ? check_qvar_types(t, Jtot)
                      : payoffs == ChainTypes::kGamma ? check_gamma_types(t, Jtot, spot) : check_fourier_types(t, Jtot, spot))
      return rc;
    dtaus.resize(M);
    double t0 = 0.0;
    for (int m = 0; m < M; ++m) {
      B200SV_REQUIRE(ttms[m] > t0, "ttms must be positive and strictly increasing");
      dtaus[m] = ttms[m] - t0;
      t0 = ttms[m];
    }
    B200SV_REQUIRE(Jtot == 0 || strikes, "null pointer");
    per_set_grid = !(vol_scaler > 0.0);
    ss.resize(std::max((size_t)B * Jtot, (size_t)1));
    if (qvar) qs.resize(std::max(Jtot, 1));
    for (int b = 0; b < B; ++b)
      for (int m = 0; m < M; ++m)
        for (int j = offsets[m]; j < offsets[m + 1]; ++j) {
          B200SV_REQUIRE(strikes[j] > 0.0, "strikes must be positive");
          ss[(size_t)b * Jtot + (j - offsets[0])] = StrikeSpec{strikes[j], forwards[m], discfactors[m], (int)types[j], b * M + m, ttms[m],
                                                               per_set_grid ? b : 0};
          if (qvar) qs[j - offsets[0]] = SumSpec{strikes[j] * ttms[m], discfactors[m], ttms[m], (int)types[j], m};
        }
    if (qvar) {                                     // utils/mgf_pricer.py:79-85: psi grid, phi = 0 (MMA) | 1 (inverse)
      build_grid(-0.5, 4000.0, P, psi);
      phi.assign(2 * (size_t)P, 0.0);
      if (!spot)
        for (int i = 0; i < P; ++i) phi[2 * i] = 1.0;
      return 0;
    }
    std::vector<double> one;
    for (int g = 0; g < (per_set_grid ? B : 1); ++g) {
      build_phi(per_set_grid ? default_vol_scaler(params[g], ttms[0]) : vol_scaler, spot, P, one);
      phi.insert(phi.end(), one.begin(), one.end());
    }
    return 0;
  }
};

// The stream, memory-pool setting and closing synchronisation of one host-level call: `return call.sync.done();`.
struct HostCall {
  cudaStream_t st = current_stream();
  StreamSync sync{st};
  HostCall() { ensure_pool_threshold(); }
};

// A prepared chain on the device: upload() queues the grid(s), psi and strike rows; the model routes add their per-maturity inputs
// (spec and the LogSV model tangents dspec, or dt), write the [B][M][P] log-MGF into lm (and A into a), and sums() prices every strike and
// copies the prices back.
struct ChainDev : HostCall {
  DevBuf phi{st}, psi{st}, rows{st}, spec{st}, dspec{st}, dt{st}, a{st}, lm{st}, pr{st}, iv{st};

  int upload(const FourierChain& c) {
    B200SV_CUDA(phi.upload(c.phi.data(), c.phi.size()));
    if (c.qvar) {
      B200SV_CUDA(psi.upload(c.psi.data(), c.psi.size()));
      B200SV_CUDA(rows.upload(c.qs.data(), c.qs.size()));
    } else {
      B200SV_CUDA(rows.upload(c.ss.data(), c.ss.size()));
    }
    B200SV_CUDA(lm.alloc(sizeof(cd) * (size_t)c.B * c.M * c.P));
    B200SV_CUDA(pr.alloc(sizeof(double) * c.ss.size()));
    return 0;
  }

  // vanilla (or Q_VAR, or with risk-premia gammas the gamma) Fourier sum, one CTA per strike; no launch on an empty chain.  gammas [G] and
  // norm_gfwd [B][M][2] (device, both or neither): the gamma of each grid and the (normaliser, gamma forward) of each slice.
  int sums(const FourierChain& c, double* prices_out, double* ivols_out, const double* gammas = nullptr, const double* norm_gfwd = nullptr) {
    if (c.Jtot == 0) return 0;
    const size_t nq = (size_t)c.B * c.Jtot;
    if (ivols_out) B200SV_CUDA(iv.alloc(sizeof(double) * nq));
    if (c.qvar)
      fourier_sum_kernel<<<(unsigned)nq, kFourierThreads, 0, st>>>(lm.as<cd>(), psi.as<cd>(), c.P, rows.as<SumSpec>(), kModeQvar, 0,
                                                                    pr.as<double>());
    else if (gammas)
      fourier_gamma_batch_kernel<<<(unsigned)nq, kFourierThreads, 0, st>>>(lm.as<cd>(), phi.as<cd>(), c.P, rows.as<StrikeSpec>(), gammas,
                                                                            norm_gfwd, pr.as<double>(), iv.as<double>());
    else
      fourier_vanilla_kernel<<<(unsigned)nq, kFourierThreads, 0, st>>>(lm.as<cd>(), phi.as<cd>(), c.P, rows.as<StrikeSpec>(), c.spot ? 1 : 0,
                                                                        1, pr.as<double>(), iv.as<double>());
    if (int rc = check_launch("fourier sum kernel")) return rc;
    B200SV_CUDA(pr.download(prices_out, nq));
    B200SV_CUDA(iv.download(ivols_out, nq));
    return 0;
  }
};

// Validation of b200sv_logsv_price_chain and its greeks, in this order: variable type, sizes, expansion order, the chain.
static int prepare_logsv_chain(FourierChain& c, const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                               const double* discfactors, const int* offsets, const double* strikes, const int8_t* types, int is_spot_measure,
                               int variable_type, int expansion_order, double vol_scaler, int P) {
  if (variable_type != B200SV_LOG_RETURN && variable_type != B200SV_Q_VAR) return fail(-4, "variable_type not implemented");   // logsv_pricer.py:733-734
  const bool qvar = variable_type == B200SV_Q_VAR;
  if (int rc = c.init(false, 1, M, P > 0 ? P : qvar ? 40000 : 1000, offsets)) return rc;   // utils/mgf_pricer.py:13, :44
  if (expansion_order != B200SV_ORDER_FIRST && expansion_order != B200SV_ORDER_SECOND)
    return fail(-4, "expansion_order not implemented");                    // affine_expansion.py:680-681
  return c.build(params, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure != 0,
                 qvar ? ChainTypes::kQvar : ChainTypes::kFourier, vol_scaler);
}

static int prepare_heston_chain(FourierChain& c, const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                const double* discfactors, const int* offsets, const double* strikes, const int8_t* types, int variable_type,
                                double vol_scaler, int P) {
  if (variable_type != B200SV_LOG_RETURN && variable_type != B200SV_Q_VAR) return fail(-4, "variable_type not implemented");   // heston_pricer.py:276-277
  const bool qvar = variable_type == B200SV_Q_VAR;
  if (int rc = c.init(false, 1, M, P > 0 ? P : qvar ? 40000 : 1000, offsets)) return rc;
  return c.build(params, ttms, forwards, discfactors, offsets, strikes, types, true, qvar ? ChainTypes::kQvar : ChainTypes::kFourier,
                 vol_scaler);
}

// The LogSV pricing launches of a prepared chain (single, greeks and batch routes): logsv_mgf_kernel over the B sets, then the sums.
static int queue_logsv_prices(ChainDev& d, const FourierChain& c, const b200sv_logsv_params* params, const double* etas, int N,
                              double* prices_out, double* ivols_out) {
  std::vector<ChainSpec> spec((size_t)c.B * c.M);
  std::vector<double> yb(c.B);
  for (int b = 0; b < c.B; ++b) {
    yb[b] = params[b].sigma0 - params[b].theta;
    for (int m = 0; m < c.M; ++m)
      spec[(size_t)b * c.M + m] = ChainSpec{c.dtaus[m], make_model(params[b], etas ? etas[(size_t)b * c.M + m] : 1.0, c.spot)};
  }
  DevBuf d_y(d.st);
  if (int rc = d.upload(c)) return rc;
  B200SV_CUDA(d.spec.upload(spec.data(), spec.size()));
  if (c.batch) B200SV_CUDA(d_y.upload(yb.data(), yb.size()));
  B200SV_CUDA(d.a.alloc(sizeof(cd) * (size_t)c.B * c.M * c.P * N));
  launch_logsv_mgf(N, d.st, d.phi.as<cd>(), d.psi.as<cd>(), c.P, c.M, d.spec.as<ChainSpec>(), nullptr, d.a.as<cd>(), d.lm.as<cd>(),
                   c.batch ? 0.0 : yb[0], c.B, d_y.as<double>(), c.batch && c.per_set_grid ? c.P : 0);
  if (int rc = check_launch("logsv_mgf_kernel")) return rc;
  return d.sums(c, prices_out, ivols_out);
}

// The Heston pricing launches of a prepared chain: heston_mgf_kernel (blockIdx.y = set), then the sums.
static int queue_heston_prices(ChainDev& d, const FourierChain& c, const b200sv_heston_params* params, double* prices_out, double* ivols_out) {
  DevBuf d_hp(d.st);
  if (int rc = d.upload(c)) return rc;
  B200SV_CUDA(d.dt.upload(c.dtaus.data(), c.dtaus.size()));
  if (c.batch) B200SV_CUDA(d_hp.upload(params, c.B));
  const int tpb = c.batch ? 64 : mgf_block_threads(c.P);
  heston_mgf_kernel<<<dim3((c.P + tpb - 1) / tpb, c.B), tpb, 0, d.st>>>(d.phi.as<cd>(), d.psi.as<cd>(), c.P, c.M, d.dt.as<double>(), params[0],
                                                                        nullptr, nullptr, nullptr, nullptr, d.lm.as<cd>(),
                                                                        d_hp.as<b200sv_heston_params>(), c.per_set_grid && c.batch ? c.P : 0);
  if (int rc = check_launch("heston_mgf_kernel")) return rc;
  return d.sums(c, prices_out, ivols_out);
}

// Validation of b200sv_hawkesjd_price_chain and its greeks: sizes, then the chain; the grid sits on Re = -1/2 - gamma (gamma = 0 without
// the risk kernel) under both measures -- get_transform_var_grid's default is_spot_measure=True (hawkes_jd_pricer.py:385), real_phi (:451).
static int prepare_hawkes_chain(FourierChain& c, const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                const double* discfactors, const int* offsets, const double* strikes, const int8_t* types, int is_spot_measure,
                                double vol_scaler, int P, double risk_premia_gamma) {
  const bool with_gamma = risk_premia_gamma == risk_premia_gamma;
  if (int rc = c.init(false, 1, M, P > 0 ? P : 500, offsets)) return rc;     // MAX_PHI, hawkes_jd_pricer.py:37
  if (int rc = c.build(params, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure != 0,
                       with_gamma ? ChainTypes::kGamma : ChainTypes::kFourier, vol_scaler))
    return rc;
  for (int i = 0; i < c.P; ++i) c.phi[2 * i] = with_gamma ? -0.5 - risk_premia_gamma : -0.5;
  return 0;
}

// The Hawkes pricing launches of a prepared chain (price, greeks and batch routes): the maturity increments go to d.dt, then
// hawkes_mgf_kernel carries A over the maturities, one launch per set queued back to back (a kernel of its own that read the constants per
// set from memory contracts its fp64 arithmetic into different fused multiply-adds and moves prices by an ulp, DESIGN.md §9), keeping A in
// d.a for a single set only; then the sums, the gamma slice pricer when gammas / norm_gfwd (device, see ChainDev::sums) are given.
static int queue_hawkes_prices(ChainDev& d, const FourierChain& c, const HawkesMgfConsts* k, double* prices_out, double* ivols_out = nullptr,
                               const double* gammas = nullptr, const double* norm_gfwd = nullptr) {
  if (int rc = d.upload(c)) return rc;
  B200SV_CUDA(d.dt.upload(c.dtaus.data(), c.dtaus.size()));
  if (!c.batch) B200SV_CUDA(d.a.alloc(sizeof(cd) * (size_t)c.M * c.P * 3));
  for (int b = 0; b < c.B; ++b) {
    launch_hawkes_mgf(d.st, d.phi.as<cd>() + (c.per_set_grid ? (size_t)b * c.P : 0), nullptr, c.P, c.M, d.dt.as<double>(), k[b], nullptr,
                      d.a.as<cd>(), d.lm.as<cd>() + (size_t)b * c.M * c.P, 0);
    if (int rc = check_launch("hawkes_mgf_kernel")) return rc;
  }
  return d.sums(c, prices_out, ivols_out, gammas, norm_gfwd);
}

// The (normaliser, gamma forward) of one slice from its two restarted log-MGFs lm2 [2] (complex: lm2[0] at -gamma, lm2[2] at -gamma - 1):
// ng = (1 / e^{lm(-gamma)}, forward e^{lm(-gamma - 1)} / e^{lm(-gamma)}).  On the host, where every route that prices under the risk kernel
// forms it, so that they all get the same bits.
static void risk_kernel_slice(const double* lm2, double forward, double* ng) {
  ng[0] = 1.0 / std::exp(lm2[0]);
  ng[1] = forward * std::exp(lm2[2]) * ng[0];
}

// hawkesjd_forwards_under_risk_kernel (:487-515) for B parameter sets k[B] under gammas[B]: two single-point solves per (set, maturity) at
// phi = -gamma and -gamma - 1, each restarted from A = 0 and integrated over the full maturity ttms[m]; one copy back, then on the host
// ng [B][M][2] = risk_kernel_slice of each (set, maturity).
static int risk_kernel_normalizers(cudaStream_t st, const HawkesMgfConsts* k, const double* gammas, int B, int M, const double* ttms,
                                   const double* forwards, std::vector<double>& ng) {
  std::vector<double> two(4 * (size_t)B, 0.0), lm2(4 * (size_t)B * M);
  for (int b = 0; b < B; ++b) {
    two[4 * (size_t)b] = -gammas[b];
    two[4 * (size_t)b + 2] = -gammas[b] - 1.0;
  }
  DevBuf d_ttm(st), d_two(st), d_lm2(st);
  B200SV_CUDA(d_ttm.upload(ttms, M));
  B200SV_CUDA(d_two.upload(cplx(two.data()), 2 * (size_t)B));
  B200SV_CUDA(d_lm2.alloc(sizeof(cd) * 2 * (size_t)B * M));
  for (int b = 0; b < B; ++b) {
    launch_hawkes_mgf(st, d_two.as<cd>() + 2 * b, nullptr, 2, M, d_ttm.as<double>(), k[b], nullptr, nullptr, d_lm2.as<cd>() + 2 * (size_t)M * b, 1);
    if (int rc = check_launch("hawkes_mgf_kernel")) return rc;
  }
  B200SV_CUDA(d_lm2.download(cplx(lm2.data()), 2 * (size_t)B * M));
  B200SV_CUDA(cudaStreamSynchronize(st));
  ng.resize(2 * (size_t)B * M);
  for (int b = 0; b < B; ++b)
    for (int m = 0; m < M; ++m) {                                            // log_mgf layout [b][m][point]
      const size_t s = (size_t)b * M + m;
      risk_kernel_slice(lm2.data() + 4 * s, forwards[m], ng.data() + 2 * s);
    }
  return 0;
}

// The Re phi of the grids of a built batch chain (prepare_hawkes_batch, and each group of b200sv_hawkesjd_price_chains_batch_gamma).
static void hawkes_batch_grids(FourierChain& c, const double* gammas) {
  const int B = c.B;
  if (gammas && !c.per_set_grid) {
    const std::vector<double> one(c.phi);
    for (int b = 1; b < B; ++b) c.phi.insert(c.phi.end(), one.begin(), one.end());
    for (size_t i = 0; i < c.ss.size(); ++i) c.ss[i].grid = (int)(i / c.Jtot);
    c.per_set_grid = true;
  }
  for (int g = 0; g < (c.per_set_grid ? B : 1); ++g)
    for (int i = 0; i < c.P; ++i) c.phi[2 * ((size_t)g * c.P + i)] = gammas ? -0.5 - gammas[g] : -0.5;
}

// Validation of b200sv_hawkesjd_price_chain_batch: sizes, the risk-premia gammas (all finite), then the chain.  The grids follow
// prepare_hawkes_chain set by set: Re phi = -1/2 - gamma_b under both measures.  With gammas every set needs its own grid even when
// vol_scaler pins the imaginary parts, since the real parts differ.
static int prepare_hawkes_batch(FourierChain& c, const b200sv_hawkes_params* params, int B, int M, const double* ttms, const double* forwards,
                                const double* discfactors, const int* offsets, const double* strikes, const int8_t* types, int is_spot_measure,
                                double vol_scaler, int P, const double* gammas) {
  if (int rc = c.init(true, B, M, P > 0 ? P : 500, offsets)) return rc;     // MAX_PHI, hawkes_jd_pricer.py:37
  if (gammas)
    for (int b = 0; b < B; ++b) B200SV_REQUIRE(std::isfinite(gammas[b]), "gammas must be finite (NULL: no risk kernel)");
  if (int rc = c.build(params, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure != 0,
                       gammas ? ChainTypes::kGamma : ChainTypes::kFourier, vol_scaler))
    return rc;
  hawkes_batch_grids(c, gammas);
  return 0;
}

// Plumbing of the single-grid entry points: phi [P], psi [P] (when given) and a_in [P][n] (when given) go up, `launch` queues its
// kernel(s) on them and returns check_launch's code, then a_out [P][n] and log_mgf_out [P] (when given) come back.
template <class Launch>
static int run_grid(const double* phi, const double* psi, int P, const double* a_in, int n, double* a_out, double* log_mgf_out, Launch launch) {
  HostCall call;
  const cudaStream_t st = call.st;
  DevBuf d_phi(st), d_psi(st), d_a0(st), d_a1(st), d_lm(st);
  const size_t na = (size_t)P * n;
  B200SV_CUDA(d_phi.upload(cplx(phi), P));
  if (psi) B200SV_CUDA(d_psi.upload(cplx(psi), P));
  if (a_in) B200SV_CUDA(d_a0.upload(cplx(a_in), na));
  if (a_out) B200SV_CUDA(d_a1.alloc(sizeof(cd) * na));
  if (log_mgf_out) B200SV_CUDA(d_lm.alloc(sizeof(cd) * P));
  if (int rc = launch(st, d_phi.as<cd>(), d_psi.as<cd>(), d_a0.as<cd>(), d_a1.as<cd>(), d_lm.as<cd>())) return rc;
  B200SV_CUDA(d_a1.download(cplx(a_out), na));
  B200SV_CUDA(d_lm.download(cplx(log_mgf_out), P));
  return call.sync.done();
}

// One CTA per strike over a caller-supplied log-MGF and grid (b200sv_fourier_*): log_mgf, grid and the rows go up, `launch` queues the sum
// kernel and returns check_launch's code, the J results come back.
template <class Row, class Launch>
static int run_sums(const double* log_mgf, const double* grid, int P, const std::vector<Row>& rows, double* out, Launch launch) {
  HostCall call;
  const cudaStream_t st = call.st;
  DevBuf d_g(st), d_lm(st), d_rows(st), d_out(st);
  B200SV_CUDA(d_g.upload(cplx(grid), P));
  B200SV_CUDA(d_lm.upload(cplx(log_mgf), P));
  B200SV_CUDA(d_rows.upload(rows.data(), rows.size()));
  B200SV_CUDA(d_out.alloc(sizeof(double) * rows.size()));
  if (int rc = launch(st, (unsigned)rows.size(), d_lm.as<cd>(), d_g.as<cd>(), d_rows.as<Row>(), d_out.as<double>())) return rc;
  B200SV_CUDA(d_out.download(out, rows.size()));
  return call.sync.done();
}

static int fourier_sum_host(const double* log_mgf, const double* grid, int P, const std::vector<SumSpec>& specs, int mode, int all_calls,
                            double* out) {
  return run_sums(log_mgf, grid, P, specs, out, [&](cudaStream_t st, unsigned J, const cd* lm, const cd* g, const SumSpec* ss, double* pr) {
    fourier_sum_kernel<<<J, kFourierThreads, 0, st>>>(lm, g, P, ss, mode, all_calls, pr);
    return check_launch("fourier_sum_kernel");
  });
}

// The first-order Fourier sums of a prepared chain (b200sv_*_price_chain_greeks, and the LogSV / Heston _hessian): the tangent kernel
// writes dlm [NP][M][P] (and, for LogSV and Hawkes, its own primal log-MGF lm [M][P] and nfev [P]); sums() queues
// fourier_vanilla_greeks_kernel on the log-MGF it is given, and dlm and the greeks [2 + NP][J] stay on the device for the launches that
// follow; download() queues the copies and synchronises.
template <int NP>
struct GreeksDev {
  DevBuf dlm, lm, nfev, g;
  explicit GreeksDev(cudaStream_t s) : dlm(s), lm(s), nfev(s), g(s) {}

  int alloc(const FourierChain& c, bool primal) {
    B200SV_CUDA(dlm.alloc(sizeof(cd) * (size_t)NP * c.M * c.P));
    if (primal) {
      B200SV_CUDA(lm.alloc(sizeof(cd) * (size_t)c.M * c.P));
      B200SV_CUDA(nfev.alloc(sizeof(int) * c.P));
    }
    B200SV_CUDA(g.alloc(sizeof(double) * (size_t)(2 + NP) * c.ss.size()));
    return 0;
  }
  // no launch on an empty chain
  int sums(const ChainDev& d, const FourierChain& c, const cd* log_mgf) {
    if (c.Jtot == 0) return 0;
    fourier_vanilla_greeks_kernel<NP><<<c.Jtot, kFourierThreads, 0, d.st>>>(log_mgf, dlm.as<cd>(), d.phi.as<cd>(), c.P, c.M,
                                                                            d.rows.as<StrikeSpec>(), c.spot ? 1 : 0, g.as<double>());
    return check_launch("fourier_vanilla_greeks_kernel");
  }
  int download(ChainDev& d, const FourierChain& c, double* greeks_out, double* dlog_mgf_out, int* nfev_out) {
    if (c.Jtot > 0) B200SV_CUDA(g.download(greeks_out, (size_t)(2 + NP) * c.Jtot));
    B200SV_CUDA(dlm.download(cplx(dlog_mgf_out), (size_t)NP * c.M * c.P));
    B200SV_CUDA(nfev.download(nfev_out, c.P));
    return d.sync.done();
  }
};

// The first-order sensitivity launches of a prepared LogSV chain: the pricing launches, logsv_mgf_tangent_kernel on the model tangents
// d.dspec (which the Hessian kernel reads too), then the sums on the tangent kernel's own primal log-MGF (DESIGN.md §4.2).
static int queue_logsv_greeks(ChainDev& d, GreeksDev<1 + kLogsvOdeDirs>& t, const FourierChain& c, const b200sv_logsv_params* params,
                              const double* etas, int expansion_order, double* prices_out) {
  const int N = expansion_order == B200SV_ORDER_FIRST ? 3 : 5, M = c.M, P = c.P;
  std::vector<LogsvModelTangent> dspec((size_t)M * kLogsvOdeDirs);
  for (int m = 0; m < M; ++m) {
    LogsvModelTangent tg[kLogsvOdeDirs];
    make_model_tangents(*params, etas ? etas[m] : 1.0, c.spot, tg);
    std::copy(tg, tg + kLogsvOdeDirs, dspec.begin() + (size_t)m * kLogsvOdeDirs);
  }
  if (int rc = queue_logsv_prices(d, c, params, etas, N, prices_out, nullptr)) return rc;
  B200SV_CUDA(d.dspec.upload(dspec.data(), dspec.size()));
  if (int rc = t.alloc(c, true)) return rc;
  const auto tangent = N == 5 ? logsv_mgf_tangent_kernel<5> : logsv_mgf_tangent_kernel<3>;
  tangent<<<(P * kLogsvOdeDirs + kTangentTPB - 1) / kTangentTPB, kTangentTPB, 0, d.st>>>(d.phi.as<cd>(), P, M, d.spec.as<ChainSpec>(),
                                                                                       d.dspec.as<LogsvModelTangent>(),
                                                                                       params->sigma0 - params->theta, t.dlm.as<cd>(),
                                                                                       t.lm.as<cd>(), nullptr, t.nfev.as<int>());
  if (int rc = check_launch("logsv_mgf_tangent_kernel")) return rc;
  return t.sums(d, c, t.lm.as<cd>());
}

// The Heston twin: the pricing launches, heston_mgf_tangent_kernel, then the sums on the pricing launch's log-MGF (heston_mgf_kernel is a
// per-thread closed form, the same for any block size).
static int queue_heston_greeks(ChainDev& d, GreeksDev<1 + kHestonOdeDirs>& t, const FourierChain& c, const b200sv_heston_params* params,
                               double* prices_out) {
  if (int rc = queue_heston_prices(d, c, params, prices_out, nullptr)) return rc;
  if (int rc = t.alloc(c, false)) return rc;
  heston_mgf_tangent_kernel<<<(c.P * kHestonOdeDirs + 63) / 64, 64, 0, d.st>>>(d.phi.as<cd>(), c.P, c.M, d.dt.as<double>(), *params,
                                                                               t.dlm.as<cd>());
  if (int rc = check_launch("heston_mgf_tangent_kernel")) return rc;
  return t.sums(d, c, d.lm.as<cd>());
}

// The Hawkes twin, without a risk kernel: the pricing launches, hawkes_mgf_tangent_kernel on the constants k, then the sums on the tangent
// kernel's own primal log-MGF, on the mesh the tangents were stepped on (DESIGN.md §4.3).
static int queue_hawkes_greeks(ChainDev& d, GreeksDev<kHawkesGreekParams>& t, const FourierChain& c, const b200sv_hawkes_params& params,
                               const HawkesMgfConsts& k, double* prices_out) {
  if (int rc = queue_hawkes_prices(d, c, &k, prices_out)) return rc;
  if (int rc = t.alloc(c, true)) return rc;
  launch_hawkes_mgf_tangent<false>(d.st, d.phi.as<cd>(), c.P, c.M, d.dt.as<double>(), k, make_hawkes_tangents(params), 0, t.dlm.as<cd>(),
                                   t.lm.as<cd>(), t.nfev.as<int>());
  if (int rc = check_launch("hawkes_mgf_tangent_kernel")) return rc;
  return t.sums(d, c, t.lm.as<cd>());
}

// The device side of the risk kernel's normaliser points, kept for the launches that follow the first-order ones: gamma, (normaliser, gamma
// forward) ng [M][2], the two points (-gamma, -gamma - 1), ttms [M] and the restarted tangents dn [16][M][2] (complex).
struct HawkesRpDev {
  DevBuf gam, ng, two, ttm, dn;
  explicit HawkesRpDev(cudaStream_t s) : gam(s), ng(s), two(s), ttm(s), dn(s) {}
};

// The first-order launches of b200sv_hawkesjd_price_chain_risk_premia_greeks on a prepared chain (DESIGN.md §4.12): the pricing launches of
// b200sv_hawkesjd_price_chain with the gamma (the restarted normaliser launch, its one synchronisation, the Riccati launch and the gamma
// sums: bit-identical prices), then hawkes_mgf_tangent_kernel<TPB, true> at the two normaliser points (restarted) and on the grid (carried), and
// fourier_gamma_greeks_kernel on the grid tangent kernel's own primal log-MGF (no launch on an empty chain).
static int queue_hawkes_rp_greeks(ChainDev& d, GreeksDev<kHawkesRpParams>& g, HawkesRpDev& r, const FourierChain& c,
                                  const b200sv_hawkes_params& params, const HawkesMgfConsts& k, const double* ttms, const double* forwards,
                                  double gamma, double* prices_out) {
  const int M = c.M, P = c.P;
  std::vector<double> ng;
  if (int rc = risk_kernel_normalizers(d.st, &k, &gamma, 1, M, ttms, forwards, ng)) return rc;
  B200SV_CUDA(r.gam.upload(&gamma, 1));
  B200SV_CUDA(r.ng.upload(ng.data(), ng.size()));
  if (int rc = queue_hawkes_prices(d, c, &k, prices_out, nullptr, r.gam.as<double>(), r.ng.as<double>())) return rc;
  const HawkesTangentDirs dirs = make_hawkes_tangents(params);
  const double two[4] = {-gamma, 0.0, -gamma - 1.0, 0.0};
  B200SV_CUDA(r.two.upload(cplx(two), 2));
  B200SV_CUDA(r.ttm.upload(ttms, M));
  B200SV_CUDA(r.dn.alloc(sizeof(cd) * (size_t)kHawkesRpParams * M * 2));
  launch_hawkes_mgf_tangent<true>(d.st, r.two.as<cd>(), 2, M, r.ttm.as<double>(), k, dirs, 1, r.dn.as<cd>(), nullptr, nullptr);
  if (int rc = check_launch("hawkes_mgf_tangent_kernel")) return rc;
  if (int rc = g.alloc(c, true)) return rc;
  launch_hawkes_mgf_tangent<true>(d.st, d.phi.as<cd>(), P, M, d.dt.as<double>(), k, dirs, 0, g.dlm.as<cd>(), g.lm.as<cd>(), g.nfev.as<int>());
  if (int rc = check_launch("hawkes_mgf_tangent_kernel")) return rc;
  if (c.Jtot > 0) {
    fourier_gamma_greeks_kernel<<<c.Jtot, kFourierThreads, 0, d.st>>>(g.lm.as<cd>(), g.dlm.as<cd>(), r.dn.as<cd>(), d.phi.as<cd>(), P, M,
                                                                      d.rows.as<StrikeSpec>(), gamma, r.ng.as<double>(), g.g.as<double>());
    if (int rc = check_launch("fourier_gamma_greeks_kernel")) return rc;
  }
  return 0;
}

// hawkes_mgf_hessian_kernel<Phi> at the n points phi, one thread per (point, pair), on the second field derivatives d2c (make_hawkes_hessian)
template <bool Phi>
static int launch_hawkes_mgf_hessian(cudaStream_t st, const cd* phi, int n, int M, const double* dtaus, const HawkesMgfConsts& k,
                                     const HawkesTangentDirs& dirs, const DevBuf& d2c, int restart, cd* d2lm) {
  constexpr int D = kHawkesOdeDirs + Phi, TPB = kHawkesHessianTPB;
  hawkes_mgf_hessian_kernel<Phi><<<(n * (D * (D + 1) / 2) + TPB - 1) / TPB, TPB, 0, st>>>(phi, n, M, dtaus, k, dirs, d2c.as<HawkesMgfConsts>(),
                                                                                          restart, d2lm);
  return check_launch("hawkes_mgf_hessian_kernel");
}

// The grid launch of both Hawkes Hessian entry points, after their first-order launches: make_hawkes_hessian's table for the 13 + Phi
// directions into d2c, then hawkes_mgf_hessian_kernel<Phi> carried over the grid into d2lm [NH][M][P] (NH = 120, or 136 with Phi)
template <bool Phi>
static int queue_hawkes_hessian(ChainDev& d, const FourierChain& c, const b200sv_hawkes_params& params, const HawkesMgfConsts& k,
                                const HawkesTangentDirs& dirs, DevBuf& d2c, DevBuf& d2lm) {
  constexpr int NP = kHawkesGreekParams + Phi, NH = NP * (NP + 1) / 2;
  const std::vector<HawkesMgfConsts> h = make_hawkes_hessian(params, kHawkesOdeDirs + Phi);
  B200SV_CUDA(d2c.upload(h.data(), h.size()));
  B200SV_CUDA(d2lm.alloc(sizeof(cd) * (size_t)NH * c.M * c.P));
  return launch_hawkes_mgf_hessian<Phi>(d.st, d.phi.as<cd>(), c.P, c.M, d.dt.as<double>(), k, dirs, d2c, 0, d2lm.as<cd>());
}

// The second-order sums of b200sv_*_price_chain_hessian after its Hessian kernel wrote d2lm [NH][M][P]: fourier_vanilla_hessian_kernel
// (fourier_vanilla_hessian_split_kernel for Hawkes' 15 parameters) on log_mgf and the first-order tangents dlm [NP][M][P] (no launch on an
// empty chain), then vanna, the Hessian rows and d2lm come back; the first-order outputs follow with GreeksDev::download().
template <int NP>
static int queue_hessian_sums(ChainDev& d, const FourierChain& c, const cd* log_mgf, const cd* dlm, const DevBuf& d2lm, double* vanna_out,
                              double* hessian_out, double* d2log_mgf_out) {
  constexpr int NH = NP * (NP + 1) / 2;
  DevBuf d_v(d.st), d_h(d.st);
  if (c.Jtot > 0) {
    B200SV_CUDA(d_v.alloc(sizeof(double) * (size_t)NP * c.Jtot));
    B200SV_CUDA(d_h.alloc(sizeof(double) * (size_t)NH * c.Jtot));
    if constexpr (NP <= 6) {      // LogSV, Heston: every row of a strike in one CTA
      fourier_vanilla_hessian_kernel<NP><<<c.Jtot, kFourierThreads, 0, d.st>>>(log_mgf, dlm, d2lm.as<cd>(), d.phi.as<cd>(), c.P, c.M,
                                                                               d.rows.as<StrikeSpec>(), c.spot ? 1 : 0, d_v.as<double>(),
                                                                               d_h.as<double>());
      if (int rc = check_launch("fourier_vanilla_hessian_kernel")) return rc;
    } else {                      // Hawkes: the vanna CTA and NH / NP Hessian CTAs per strike
      const dim3 grid(c.Jtot, 1 + (NH + NP - 1) / NP);
      fourier_vanilla_hessian_split_kernel<NP><<<grid, kFourierThreads, 0, d.st>>>(log_mgf, dlm, d2lm.as<cd>(), d.phi.as<cd>(), c.P, c.M,
                                                                                   d.rows.as<StrikeSpec>(), c.spot ? 1 : 0, d_v.as<double>(),
                                                                                   d_h.as<double>());
      if (int rc = check_launch("fourier_vanilla_hessian_split_kernel")) return rc;
    }
    B200SV_CUDA(d_v.download(vanna_out, (size_t)NP * c.Jtot));
    B200SV_CUDA(d_h.download(hessian_out, (size_t)NH * c.Jtot));
  }
  B200SV_CUDA(d2lm.download(cplx(d2log_mgf_out), (size_t)NH * c.M * c.P));
  return 0;
}

// The theta launches of b200sv_*_price_chain_greeks_theta after the greeks launches of the twin (whose outputs they do not touch): the
// theta kernel writes dlm [M][P] (and nfev [P] for the adaptive routes), then fourier_vanilla_greeks_kernel<1> sums it on the log-MGF the
// parameter rows were summed on: its row 2 is scale * S_T = d price / d T, so theta = -row 2 (DESIGN.md §4.8).
struct ThetaDev {
  DevBuf dlm, nfev, g;
  explicit ThetaDev(cudaStream_t s) : dlm(s), nfev(s), g(s) {}

  int alloc(const FourierChain& c, bool adaptive) {
    B200SV_CUDA(dlm.alloc(sizeof(cd) * (size_t)c.M * c.P));
    if (adaptive) B200SV_CUDA(nfev.alloc(sizeof(int) * c.P));
    B200SV_CUDA(g.alloc(sizeof(double) * 3 * c.ss.size()));
    return 0;
  }
  int sums(const ChainDev& d, const FourierChain& c, const cd* log_mgf) {
    if (int rc = check_launch("theta kernel")) return rc;
    if (c.Jtot == 0) return 0;
    fourier_vanilla_greeks_kernel<1><<<c.Jtot, kFourierThreads, 0, d.st>>>(log_mgf, dlm.as<cd>(), d.phi.as<cd>(), c.P, c.M,
                                                                           d.rows.as<StrikeSpec>(), c.spot ? 1 : 0, g.as<double>());
    return check_launch("fourier_vanilla_greeks_kernel");
  }
  // queues the copies of d price / d T into theta_out and of dlm / nfev (when asked); finish() negates after the closing synchronisation
  int download(const FourierChain& c, double* theta_out, double* dlog_mgf_theta_out, int* nfev_out) {
    if (c.Jtot > 0)
      B200SV_CUDA(cudaMemcpyAsync(theta_out, g.as<double>() + 2 * (size_t)c.Jtot, sizeof(double) * c.Jtot, cudaMemcpyDeviceToHost, g.st));
    B200SV_CUDA(dlm.download(cplx(dlog_mgf_theta_out), (size_t)c.M * c.P));
    B200SV_CUDA(nfev.download(nfev_out, c.P));
    return 0;
  }
  static void finish(const FourierChain& c, double* theta_out) {
    for (int j = 0; j < c.Jtot; ++j) theta_out[j] = -theta_out[j];
  }
};

static int check_expansion_order(int expansion_order) {
  if (expansion_order != B200SV_ORDER_FIRST && expansion_order != B200SV_ORDER_SECOND) return fail(-4, "expansion_order not implemented");
  return 0;
}

// ---- several chains in one call (b200sv_*_price_chains_batch) ----
// The sets of one chain form a group.  A group is validated by the same FourierChain code as b200sv_*_price_chain_batch on those sets
// alone and runs on exactly the launch that call would queue for its log-MGF (same kernel, block size and set mapping, all chosen from
// the group's |S_k| P), so every row equals that call's bit for bit and no warp ever mixes chains.  The groups' log-MGF launches go to
// streams forked from the call's stream, so that they run side by side; then ONE Fourier-sum launch prices every (set, strike) of the
// call, each CTA reading its own set's log-MGF rows and grid.
template <class Params>
struct ChainsCall {
  struct Group {
    int chain = 0, mat0 = 0;          // the chain, and its first entry in ttms / forwards / discfactors
    std::vector<int> sets;            // the call's sets on this chain, in call order
    std::vector<Params> params;
    std::vector<double> etas;         // [sets][M] (LogSV with etas only)
    std::vector<double> gammas;       // [sets] (Hawkes under the risk kernel only)
    FourierChain c;
    size_t slice0 = 0, grid0 = 0;     // the group's first log-MGF row [.][P] and first grid [.][P] in the call's buffers
  };
  std::vector<Group> groups;          // the chains that have sets, in chain order
  std::vector<StrikeSpec> rows;       // [sum_b J_k(b)]: set b's strikes in call order (slice / grid index the call's buffers)
  size_t slices = 0, grids = 0;

  // Ms[K]; chain k's maturities at ttms / forwards / discfactors [sum Ms[:k]], its Ms[k] + 1 offsets into strikes / types at
  // offsets [sum (Ms[:k] + 1)]; etas (may be NULL) [sum_b Ms[chain_of_set[b]]].  Every Ms[k] must be >= 1 (it places the chains
  // after k); of a chain that no set points at nothing else is read.  gammas (may be NULL) [B]: the Hawkes risk-premia gammas, each group
  // then validated and gridded as prepare_hawkes_batch does its sets, and every set on a grid of its own.
  int prepare(const Params* params, int B, const int* chain_of_set, int K, const int* Ms, const double* ttms, const double* forwards,
              const double* discfactors, const double* etas, const int* offsets, const double* strikes, const int8_t* types, bool spot,
              const double* vol_scalers, int P, const double* gammas = nullptr) {
    B200SV_REQUIRE(params && chain_of_set && Ms && ttms && forwards && discfactors && offsets && strikes && types && vol_scalers,
                   "null pointer");
    B200SV_REQUIRE(B >= 1 && K >= 1, "B >= 1, K >= 1");
    std::vector<int> mat0(K), off0(K), group_of(K, -1);
    for (int k = 0, m = 0; k < K; m += Ms[k], ++k) {
      B200SV_REQUIRE(Ms[k] >= 1, "every chain needs M >= 1");
      mat0[k] = m;
      off0[k] = m + k;
    }
    for (int b = 0; b < B; ++b) B200SV_REQUIRE(chain_of_set[b] >= 0 && chain_of_set[b] < K, "chain_of_set out of range");
    std::vector<size_t> eta0(B);
    for (int b = 0, e = 0; b < B; e += Ms[chain_of_set[b]], ++b) eta0[b] = e;
    for (int k = 0; k < K; ++k)
      for (int b = 0; b < B; ++b) {
        if (chain_of_set[b] != k) continue;
        if (group_of[k] < 0) {
          group_of[k] = (int)groups.size();
          groups.emplace_back();
          groups.back().chain = k;
          groups.back().mat0 = mat0[k];
        }
        Group& g = groups[group_of[k]];
        g.sets.push_back(b);
        g.params.push_back(params[b]);
        if (etas) g.etas.insert(g.etas.end(), etas + eta0[b], etas + eta0[b] + Ms[k]);
        if (gammas) g.gammas.push_back(gammas[b]);
      }
    for (Group& g : groups) {
      const int k = g.chain, m0 = g.mat0, *off = offsets + off0[k];
      if (int rc = g.c.init(true, (int)g.sets.size(), Ms[k], P > 0 ? P : 1000, off)) return rc;
      for (double y : g.gammas) B200SV_REQUIRE(std::isfinite(y), "gammas must be finite (NULL: no risk kernel)");
      if (int rc = g.c.build(g.params.data(), ttms + m0, forwards + m0, discfactors + m0, off, strikes, types, spot,
                             gammas ? ChainTypes::kGamma : ChainTypes::kFourier, vol_scalers[k]))
        return rc;
      if (gammas) hawkes_batch_grids(g.c, g.gammas.data());
      g.slice0 = slices;
      g.grid0 = grids;
      slices += (size_t)g.c.B * g.c.M;
      grids += g.c.phi.size() / (2 * (size_t)g.c.P);
    }
    std::vector<int> index(B);                // position of each set within its group
    for (const Group& g : groups)
      for (size_t i = 0; i < g.sets.size(); ++i) index[g.sets[i]] = (int)i;
    for (int b = 0; b < B; ++b) {
      const Group& g = groups[group_of[chain_of_set[b]]];
      for (int j = 0; j < g.c.Jtot; ++j) {
        StrikeSpec s = g.c.ss[(size_t)index[b] * g.c.Jtot + j];
        s.slice += (int)g.slice0;
        s.grid += (int)g.grid0;
        rows.push_back(s);
      }
    }
    return 0;
  }

  int P() const { return groups[0].c.P; }
  std::vector<double> phi() const {
    std::vector<double> all;
    for (const Group& g : groups) all.insert(all.end(), g.c.phi.begin(), g.c.phi.end());
    return all;
  }
};

// Streams forked from `st` and joined back into it: n = 1 is `st` itself, more are taken from a process-wide pool per device, created on
// first use and kept (creating them cost more than a small call's launches).  The destructor joins (if join() did not), so that the call's
// stream-ordered frees and its closing synchronisation come after every forked launch.  Two calls that share a pooled stream only wait
// for each other.
class ForkedStreams {
 public:
  ForkedStreams(cudaStream_t st, int n) : st_(st) {
    if (n <= 1) {
      s_.push_back(st);
      return;
    }
    if ((err_ = pooled(n, s_)) != cudaSuccess) return;
    cudaEvent_t e;
    if ((err_ = cudaEventCreateWithFlags(&e, cudaEventDisableTiming)) != cudaSuccess) return;
    ev_.push_back(e);
    if ((err_ = cudaEventRecord(e, st)) != cudaSuccess) return;
    for (cudaStream_t s : s_)
      if ((err_ = cudaStreamWaitEvent(s, e, 0)) != cudaSuccess) return;
    forked_ = true;
  }
  ForkedStreams(const ForkedStreams&) = delete;
  ForkedStreams& operator=(const ForkedStreams&) = delete;
  cudaError_t error() const { return err_; }
  cudaStream_t operator[](size_t i) const { return s_[i % s_.size()]; }
  cudaError_t join() {
    if (!forked_) return err_;
    forked_ = false;
    for (cudaStream_t s : s_) {
      cudaEvent_t e;
      cudaError_t rc = cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
      if (rc == cudaSuccess) {
        ev_.push_back(e);
        rc = cudaEventRecord(e, s);
      }
      if (rc == cudaSuccess) rc = cudaStreamWaitEvent(st_, e, 0);
      if (rc != cudaSuccess) {
        cudaStreamSynchronize(s);          // st_ could not be ordered after s: wait for it here
        if (err_ == cudaSuccess) err_ = rc;
      }
    }
    return err_;
  }
  ~ForkedStreams() {
    join();
    for (cudaEvent_t e : ev_) cudaEventDestroy(e);      // released once the waits on them are done
  }

 private:
  static cudaError_t pooled(int n, std::vector<cudaStream_t>& out) {
    static std::mutex mu;
    static std::vector<std::vector<cudaStream_t>> pool;   // [device]
    int dev = 0;
    if (cudaError_t e = cudaGetDevice(&dev)) return e;
    std::lock_guard<std::mutex> lock(mu);
    if ((int)pool.size() <= dev) pool.resize(dev + 1);
    std::vector<cudaStream_t>& p = pool[dev];
    while ((int)p.size() < n) {
      cudaStream_t s;
      if (cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)) return e;
      p.push_back(s);
    }
    out.assign(p.begin(), p.begin() + n);
    return cudaSuccess;
  }

  cudaStream_t st_;
  std::vector<cudaStream_t> s_;
  std::vector<cudaEvent_t> ev_;
  cudaError_t err_ = cudaSuccess;
  bool forked_ = false;
};

constexpr int kChainsStreams = 16;   // concurrent log-MGF launches of a multi-chain call (H100 runs up to 128 kernels at once)

// The device side of a prepared multi-chain call on host.st: grids and strike rows up, `per_group(g, stream, phi, lm)` queues group g's
// log-MGF launch on a forked stream (reading its grids at phi, writing its [B_k][M_k][P] rows at lm), then the one Fourier-sum launch and
// the copies back.  gammas [grids] and norm_gfwd [slices][2] (device, both or neither): the risk kernel's gamma of each grid and
// (normaliser, gamma forward) of each slice, priced by the gamma slice pricer (ChainDev::sums).
template <class Params, class PerGroup>
static int run_chains(HostCall& host, const ChainsCall<Params>& call, int is_spot, double* prices_out, double* ivols_out, PerGroup per_group,
                      const double* gammas = nullptr, const double* norm_gfwd = nullptr) {
  const cudaStream_t st = host.st;
  const int P = call.P();
  const size_t nq = call.rows.size();
  const std::vector<double> phi = call.phi();
  DevBuf d_phi(st), d_rows(st), d_lm(st), d_pr(st), d_iv(st);
  B200SV_CUDA(d_phi.upload(cplx(phi.data()), phi.size() / 2));
  B200SV_CUDA(d_rows.upload(call.rows.data(), nq));
  B200SV_CUDA(d_lm.alloc(sizeof(cd) * call.slices * P));
  B200SV_CUDA(d_pr.alloc(sizeof(double) * nq));
  if (ivols_out) B200SV_CUDA(d_iv.alloc(sizeof(double) * nq));
  {
    ForkedStreams fork(st, (int)std::min<size_t>(call.groups.size(), kChainsStreams));
    B200SV_CUDA(fork.error());
    for (size_t g = 0; g < call.groups.size(); ++g)
      if (int rc = per_group(call.groups[g], fork[g], d_phi.as<cd>() + call.groups[g].grid0 * P, d_lm.as<cd>() + call.groups[g].slice0 * P))
        return rc;
    B200SV_CUDA(fork.join());
  }
  if (gammas)
    fourier_gamma_batch_kernel<<<(unsigned)nq, kFourierThreads, 0, st>>>(d_lm.as<cd>(), d_phi.as<cd>(), P, d_rows.as<StrikeSpec>(), gammas,
                                                                          norm_gfwd, d_pr.as<double>(), d_iv.as<double>());
  else
    fourier_vanilla_kernel<<<(unsigned)nq, kFourierThreads, 0, st>>>(d_lm.as<cd>(), d_phi.as<cd>(), P, d_rows.as<StrikeSpec>(), is_spot, 1,
                                                                      d_pr.as<double>(), d_iv.as<double>());
  if (int rc = check_launch("fourier sum kernel")) return rc;
  B200SV_CUDA(d_pr.download(prices_out, nq));
  B200SV_CUDA(d_iv.download(ivols_out, nq));
  return host.sync.done();
}

}  // namespace b200sv

using namespace b200sv;

extern "C" {

int b200sv_logsv_price_chain(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                             const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                             const int8_t* types, int is_spot_measure, int variable_type, int expansion_order,
                             double vol_scaler, int P, double* prices_out, double* a_out, double* log_mgf_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out, "null pointer");
  FourierChain c;
  if (int rc = prepare_logsv_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure, variable_type,
                                   expansion_order, vol_scaler, P))
    return rc;
  const int N = expansion_order == B200SV_ORDER_FIRST ? 3 : 5;
  ChainDev d;
  if (int rc = queue_logsv_prices(d, c, params, etas, N, prices_out, nullptr)) return rc;
  B200SV_CUDA(d.a.download(cplx(a_out), (size_t)M * c.P * N));
  B200SV_CUDA(d.lm.download(cplx(log_mgf_out), (size_t)M * c.P));
  return d.sync.done();
}

int b200sv_heston_price_chain(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                              const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                              int variable_type, double vol_scaler, int P, double* prices_out, double* log_mgf_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out, "null pointer");
  FourierChain c;
  if (int rc = prepare_heston_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, variable_type, vol_scaler, P)) return rc;
  ChainDev d;
  if (int rc = queue_heston_prices(d, c, params, prices_out, nullptr)) return rc;
  B200SV_CUDA(d.lm.download(cplx(log_mgf_out), (size_t)M * c.P));
  return d.sync.done();
}

/* ---- forward-mode sensitivities of the two Fourier chain pricers (DESIGN.md §4.2) ----
 * One prepared chain: the pricing launches of b200sv_*_price_chain (same function, so bit-identical prices), then the tangent kernel and
 * fourier_vanilla_greeks_kernel, which assembles delta, gamma and the parameter rows; one synchronisation at the end. */
int b200sv_logsv_price_chain_greeks(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                    const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                    const int8_t* types, int is_spot_measure, int variable_type, int expansion_order,
                                    double vol_scaler, int P, double* prices_out, double* greeks_out, double* dlog_mgf_out,
                                    int* nfev_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && greeks_out, "null pointer");
  if (variable_type != B200SV_LOG_RETURN) return fail(-4, "variable_type not implemented: sensitivities cover LOG_RETURN only");
  FourierChain c;
  if (int rc = prepare_logsv_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure, variable_type,
                                   expansion_order, vol_scaler, P))
    return rc;
  ChainDev d;
  GreeksDev<1 + kLogsvOdeDirs> g(d.st);
  if (int rc = queue_logsv_greeks(d, g, c, params, etas, expansion_order, prices_out)) return rc;
  return g.download(d, c, greeks_out, dlog_mgf_out, nfev_out);
}

int b200sv_heston_price_chain_greeks(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                     const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                     int variable_type, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                     double* dlog_mgf_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && greeks_out, "null pointer");
  if (variable_type != B200SV_LOG_RETURN) return fail(-4, "variable_type not implemented: sensitivities cover LOG_RETURN only");
  FourierChain c;
  if (int rc = prepare_heston_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, variable_type, vol_scaler, P)) return rc;
  ChainDev d;
  GreeksDev<1 + kHestonOdeDirs> g(d.st);
  if (int rc = queue_heston_greeks(d, g, c, params, prices_out)) return rc;
  return g.download(d, c, greeks_out, dlog_mgf_out, nullptr);
}

/* ---- second-order forward-mode sensitivities of the two Fourier chain pricers (DESIGN.md §4.4) ----
 * The launches of b200sv_*_price_chain_greeks unchanged (bit-identical first-order outputs), then the Hessian kernel and
 * fourier_vanilla_hessian_kernel; one synchronisation at the end. */
int b200sv_logsv_price_chain_hessian(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                     const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                     const int8_t* types, int is_spot_measure, int variable_type, int expansion_order,
                                     double vol_scaler, int P, double* prices_out, double* greeks_out, double* dlog_mgf_out,
                                     int* nfev_out, double* vanna_out, double* hessian_out, double* d2log_mgf_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && greeks_out && vanna_out && hessian_out, "null pointer");
  if (variable_type != B200SV_LOG_RETURN) return fail(-4, "variable_type not implemented: sensitivities cover LOG_RETURN only");
  FourierChain c;
  if (int rc = prepare_logsv_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure, variable_type,
                                   expansion_order, vol_scaler, P))
    return rc;
  ChainDev d;
  GreeksDev<1 + kLogsvOdeDirs> g(d.st);
  if (int rc = queue_logsv_greeks(d, g, c, params, etas, expansion_order, prices_out)) return rc;
  const int N = expansion_order == B200SV_ORDER_FIRST ? 3 : 5, NP = 1 + kLogsvOdeDirs, NH = NP * (NP + 1) / 2;
  P = c.P;
  std::vector<LogsvModelTangent> d2spec((size_t)M * kLogsvOdePairs);
  for (int m = 0; m < M; ++m) {
    LogsvModelTangent h[kLogsvOdePairs];
    make_model_hessian(*params, etas ? etas[m] : 1.0, c.spot, h);
    std::copy(h, h + kLogsvOdePairs, d2spec.begin() + (size_t)m * kLogsvOdePairs);
  }
  DevBuf d_d2spec(d.st), d_d2lm(d.st);
  B200SV_CUDA(d_d2spec.upload(d2spec.data(), d2spec.size()));
  B200SV_CUDA(d_d2lm.alloc(sizeof(cd) * (size_t)NH * M * P));
  const auto hessian = N == 5 ? logsv_mgf_hessian_kernel<5> : logsv_mgf_hessian_kernel<3>;
  hessian<<<(P * kLogsvOdePairs + kHessianTPB - 1) / kHessianTPB, kHessianTPB, 0, d.st>>>(d.phi.as<cd>(), P, M, d.spec.as<ChainSpec>(),
                                                                                        d.dspec.as<LogsvModelTangent>(),
                                                                                        d_d2spec.as<LogsvModelTangent>(),
                                                                                        params->sigma0 - params->theta, d_d2lm.as<cd>());
  if (int rc = check_launch("logsv_mgf_hessian_kernel")) return rc;
  // the tangent kernel's primal log-MGF and tangents, as for the first-order rows
  if (int rc = queue_hessian_sums<NP>(d, c, g.lm.as<cd>(), g.dlm.as<cd>(), d_d2lm, vanna_out, hessian_out, d2log_mgf_out)) return rc;
  return g.download(d, c, greeks_out, dlog_mgf_out, nfev_out);
}

int b200sv_heston_price_chain_hessian(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                      const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                      int variable_type, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                      double* dlog_mgf_out, double* vanna_out, double* hessian_out, double* d2log_mgf_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && greeks_out && vanna_out && hessian_out, "null pointer");
  if (variable_type != B200SV_LOG_RETURN) return fail(-4, "variable_type not implemented: sensitivities cover LOG_RETURN only");
  FourierChain c;
  if (int rc = prepare_heston_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, variable_type, vol_scaler, P)) return rc;
  ChainDev d;
  GreeksDev<1 + kHestonOdeDirs> g(d.st);
  if (int rc = queue_heston_greeks(d, g, c, params, prices_out)) return rc;
  const int NP = 1 + kHestonOdeDirs, NH = NP * (NP + 1) / 2;
  P = c.P;
  DevBuf d_d2lm(d.st);
  B200SV_CUDA(d_d2lm.alloc(sizeof(cd) * (size_t)NH * M * P));
  heston_mgf_hessian_kernel<<<(P * kHestonOdePairs + 63) / 64, 64, 0, d.st>>>(d.phi.as<cd>(), P, M, d.dt.as<double>(), *params, d_d2lm.as<cd>());
  if (int rc = check_launch("heston_mgf_hessian_kernel")) return rc;
  if (int rc = queue_hessian_sums<NP>(d, c, d.lm.as<cd>(), g.dlm.as<cd>(), d_d2lm, vanna_out, hessian_out, d2log_mgf_out)) return rc;
  return g.download(d, c, greeks_out, dlog_mgf_out, nullptr);
}

/* ---- batched chain pricers: B parameter sets on one chain in one pass (calibration objective + its finite-difference gradient) ----
 * vol_scaler <= 0: each set gets its own grid from its default scaler */
int b200sv_logsv_price_chain_batch(const b200sv_logsv_params* params, int B, int M, const double* ttms, const double* forwards,
                                   const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                   const int8_t* types, int is_spot_measure, int expansion_order, double vol_scaler, int P,
                                   double* prices_out, double* ivols_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && strikes && types && prices_out, "null pointer");
  if (expansion_order != B200SV_ORDER_FIRST && expansion_order != B200SV_ORDER_SECOND) return fail(-4, "expansion_order not implemented");
  FourierChain c;
  if (int rc = c.init(true, B, M, P > 0 ? P : 1000, offsets)) return rc;
  if (int rc = c.build(params, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure != 0, ChainTypes::kFourier, vol_scaler))
    return rc;
  ChainDev d;
  if (int rc = queue_logsv_prices(d, c, params, etas, expansion_order == B200SV_ORDER_FIRST ? 3 : 5, prices_out, ivols_out)) return rc;
  return d.sync.done();
}

int b200sv_heston_price_chain_batch(const b200sv_heston_params* params, int B, int M, const double* ttms, const double* forwards,
                                    const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                    double vol_scaler, int P, double* prices_out, double* ivols_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && strikes && types && prices_out, "null pointer");
  FourierChain c;
  if (int rc = c.init(true, B, M, P > 0 ? P : 1000, offsets)) return rc;
  if (int rc = c.build(params, ttms, forwards, discfactors, offsets, strikes, types, true, ChainTypes::kFourier, vol_scaler)) return rc;
  ChainDev d;
  if (int rc = queue_heston_prices(d, c, params, prices_out, ivols_out)) return rc;
  return d.sync.done();
}

/* ---- batched chain pricers over several chains: B parameter sets, set b on chain chain_of_set[b], in one call ---- */
int b200sv_logsv_price_chains_batch(const b200sv_logsv_params* params, int B, const int* chain_of_set, int K, const int* Ms,
                                    const double* ttms, const double* forwards, const double* discfactors, const double* etas,
                                    const int* offsets, const double* strikes, const int8_t* types, int is_spot_measure, int expansion_order,
                                    const double* vol_scalers, int P, double* prices_out, double* ivols_out) {
  B200SV_REQUIRE(prices_out, "null pointer");
  if (expansion_order != B200SV_ORDER_FIRST && expansion_order != B200SV_ORDER_SECOND) return fail(-4, "expansion_order not implemented");
  const int N = expansion_order == B200SV_ORDER_FIRST ? 3 : 5;
  ChainsCall<b200sv_logsv_params> call;
  if (int rc = call.prepare(params, B, chain_of_set, K, Ms, ttms, forwards, discfactors, etas, offsets, strikes, types, is_spot_measure != 0,
                            vol_scalers, P))
    return rc;
  // per-group model inputs as queue_logsv_prices builds them: spec [B_k][M_k], yb [B_k]
  std::vector<ChainSpec> spec;
  std::vector<double> yb;
  std::vector<size_t> spec0, a0;
  size_t na = 0;
  for (const auto& g : call.groups) {
    spec0.push_back(spec.size());
    a0.push_back(na);
    na += (size_t)g.c.B * g.c.M * g.c.P * N;
    for (int b = 0; b < g.c.B; ++b) {
      yb.push_back(g.params[b].sigma0 - g.params[b].theta);
      for (int m = 0; m < g.c.M; ++m)
        spec.push_back(ChainSpec{g.c.dtaus[m], make_model(g.params[b], g.etas.empty() ? 1.0 : g.etas[(size_t)b * g.c.M + m], g.c.spot)});
    }
  }
  HostCall host;
  DevBuf d_spec(host.st), d_y(host.st), d_a(host.st);
  B200SV_CUDA(d_spec.upload(spec.data(), spec.size()));
  B200SV_CUDA(d_y.upload(yb.data(), yb.size()));
  B200SV_CUDA(d_a.alloc(sizeof(cd) * na));
  size_t gi = 0, y0 = 0;
  return run_chains(host, call, is_spot_measure != 0 ? 1 : 0, prices_out, ivols_out, [&](const auto& g, cudaStream_t s, const cd* phi, cd* lm) {
    launch_logsv_mgf(N, s, phi, nullptr, g.c.P, g.c.M, d_spec.as<ChainSpec>() + spec0[gi], nullptr, d_a.as<cd>() + a0[gi], lm, 0.0, g.c.B,
                     d_y.as<double>() + y0, g.c.per_set_grid ? g.c.P : 0);
    ++gi;
    y0 += g.c.B;
    return check_launch("logsv_mgf_kernel");
  });
}

int b200sv_heston_price_chains_batch(const b200sv_heston_params* params, int B, const int* chain_of_set, int K, const int* Ms,
                                     const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                     const double* strikes, const int8_t* types, const double* vol_scalers, int P, double* prices_out,
                                     double* ivols_out) {
  B200SV_REQUIRE(prices_out, "null pointer");
  ChainsCall<b200sv_heston_params> call;
  if (int rc = call.prepare(params, B, chain_of_set, K, Ms, ttms, forwards, discfactors, nullptr, offsets, strikes, types, true, vol_scalers, P))
    return rc;
  std::vector<double> dt;
  std::vector<b200sv_heston_params> hp;
  std::vector<size_t> dt0, hp0;
  for (const auto& g : call.groups) {
    dt0.push_back(dt.size());
    hp0.push_back(hp.size());
    dt.insert(dt.end(), g.c.dtaus.begin(), g.c.dtaus.end());
    hp.insert(hp.end(), g.params.begin(), g.params.end());
  }
  HostCall host;
  DevBuf d_dt(host.st), d_hp(host.st);
  B200SV_CUDA(d_dt.upload(dt.data(), dt.size()));
  B200SV_CUDA(d_hp.upload(hp.data(), hp.size()));
  size_t gi = 0;
  return run_chains(host, call, 1, prices_out, ivols_out, [&](const auto& g, cudaStream_t s, const cd* phi, cd* lm) {
    // queue_heston_prices' batch launch: 64 threads, blockIdx.y = set
    heston_mgf_kernel<<<dim3((g.c.P + 63) / 64, g.c.B), 64, 0, s>>>(phi, nullptr, g.c.P, g.c.M, d_dt.as<double>() + dt0[gi], g.params[0], nullptr,
                                                                    nullptr, nullptr, nullptr, lm, d_hp.as<b200sv_heston_params>() + hp0[gi],
                                                                    g.c.per_set_grid ? g.c.P : 0);
    ++gi;
    return check_launch("heston_mgf_kernel");
  });
}

// The Hawkes twin without a risk kernel: each group is validated as b200sv_hawkesjd_price_chain_batch validates its sets (default P =
// 500, Re phi = -1/2 under both measures) and integrated by ONE hawkes_mgf_sets_kernel launch, whose rows equal the single-set
// hawkes_mgf_kernel launches of that call bit for bit.
int b200sv_hawkesjd_price_chains_batch(const b200sv_hawkes_params* params, int B, const int* chain_of_set, int K, const int* Ms,
                                       const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                       const double* strikes, const int8_t* types, int is_spot_measure, const double* vol_scalers, int P,
                                       double* prices_out, double* ivols_out) {
  B200SV_REQUIRE(prices_out, "null pointer");
  ChainsCall<b200sv_hawkes_params> call;
  if (int rc = call.prepare(params, B, chain_of_set, K, Ms, ttms, forwards, discfactors, nullptr, offsets, strikes, types, is_spot_measure != 0,
                            vol_scalers, P > 0 ? P : 500))                // MAX_PHI, hawkes_jd_pricer.py:37
    return rc;
  std::vector<double> dt;
  std::vector<HawkesMgfConsts> k;
  std::vector<size_t> dt0, k0;
  for (auto& g : call.groups) {
    for (size_t i = 0; i < g.c.phi.size(); i += 2) g.c.phi[i] = -0.5;     // prepare_hawkes_batch without gammas
    dt0.push_back(dt.size());
    k0.push_back(k.size());
    dt.insert(dt.end(), g.c.dtaus.begin(), g.c.dtaus.end());
    for (const auto& p : g.params) k.push_back(make_hawkes_mgf_consts(p));
  }
  HostCall host;
  DevBuf d_dt(host.st), d_k(host.st);
  B200SV_CUDA(d_dt.upload(dt.data(), dt.size()));
  B200SV_CUDA(d_k.upload(k.data(), k.size()));
  size_t gi = 0;
  return run_chains(host, call, is_spot_measure != 0 ? 1 : 0, prices_out, ivols_out, [&](const auto& g, cudaStream_t s, const cd* phi, cd* lm) {
    launch_hawkes_mgf_sets(s, phi, g.c.P, g.c.M, d_dt.as<double>() + dt0[gi], d_k.as<HawkesMgfConsts>() + k0[gi], g.c.B,
                           g.c.per_set_grid ? g.c.P : 0, lm);
    ++gi;
    return check_launch("hawkes_mgf_sets_kernel");
  });
}

// The risk-kernel twin (DESIGN.md §4.11): gammas [B] as in b200sv_hawkesjd_price_chain_batch, each group validated and gridded as
// prepare_hawkes_batch does its sets.  ONE restarted hawkes_mgf_sets_kernel launch solves the two normaliser points of every (set,
// maturity) of the call over that maturity's full ttm; one copy back and synchronise, and risk_kernel_slice forms the (normaliser, gamma
// forward) of each slice on the host as the single-chain routes do.  Then one Riccati launch per chain and ONE gamma Fourier-sum launch.
int b200sv_hawkesjd_price_chains_batch_gamma(const b200sv_hawkes_params* params, const double* gammas, int B, const int* chain_of_set, int K,
                                             const int* Ms, const double* ttms, const double* forwards, const double* discfactors,
                                             const int* offsets, const double* strikes, const int8_t* types, int is_spot_measure,
                                             const double* vol_scalers, int P, double* prices_out, double* ivols_out) {
  B200SV_REQUIRE(gammas && prices_out, "null pointer");
  ChainsCall<b200sv_hawkes_params> call;
  if (int rc = call.prepare(params, B, chain_of_set, K, Ms, ttms, forwards, discfactors, nullptr, offsets, strikes, types, is_spot_measure != 0,
                            vol_scalers, P > 0 ? P : 500, gammas))                // MAX_PHI, hawkes_jd_pricer.py:37
    return rc;
  // Per set in grid order (the groups in chain order, a group's sets in call order): its constants, gamma, normaliser points and first
  // slice m0; per slice its ttm and forward; per group its maturity increments from dt0.
  std::vector<HawkesMgfConsts> k;
  std::vector<double> gam, two, tt, fw, dt;
  std::vector<int> m0;
  std::vector<size_t> dt0;
  for (const auto& g : call.groups) {
    dt0.push_back(dt.size());
    dt.insert(dt.end(), g.c.dtaus.begin(), g.c.dtaus.end());
    for (size_t i = 0; i < g.sets.size(); ++i) {
      k.push_back(make_hawkes_mgf_consts(g.params[i]));
      gam.push_back(g.gammas[i]);
      two.insert(two.end(), {-g.gammas[i], 0.0, -g.gammas[i] - 1.0, 0.0});
      m0.push_back((int)tt.size());
      tt.insert(tt.end(), ttms + g.mat0, ttms + g.mat0 + g.c.M);
      fw.insert(fw.end(), forwards + g.mat0, forwards + g.mat0 + g.c.M);
    }
  }
  m0.push_back((int)tt.size());
  const size_t slices = tt.size();
  HostCall host;
  DevBuf d_k(host.st), d_two(host.st), d_tt(host.st), d_m0(host.st), d_lm2(host.st), d_dt(host.st), d_gam(host.st), d_ng(host.st);
  B200SV_CUDA(d_k.upload(k.data(), k.size()));
  B200SV_CUDA(d_two.upload(cplx(two.data()), two.size() / 2));
  B200SV_CUDA(d_tt.upload(tt.data(), slices));
  B200SV_CUDA(d_m0.upload(m0.data(), m0.size()));
  B200SV_CUDA(d_lm2.alloc(sizeof(cd) * 2 * slices));
  launch_hawkes_mgf_sets<true>(host.st, d_two.as<cd>(), 2, 0, d_tt.as<double>(), d_k.as<HawkesMgfConsts>(), (int)k.size(), 2, d_lm2.as<cd>(),
                               d_m0.as<int>());
  if (int rc = check_launch("hawkes_mgf_sets_kernel")) return rc;
  std::vector<double> lm2(4 * slices), ng(2 * slices);
  B200SV_CUDA(d_lm2.download(cplx(lm2.data()), 2 * slices));
  B200SV_CUDA(cudaStreamSynchronize(host.st));
  for (size_t s = 0; s < slices; ++s) risk_kernel_slice(lm2.data() + 4 * s, fw[s], ng.data() + 2 * s);
  B200SV_CUDA(d_dt.upload(dt.data(), dt.size()));
  B200SV_CUDA(d_gam.upload(gam.data(), gam.size()));
  B200SV_CUDA(d_ng.upload(ng.data(), ng.size()));
  size_t gi = 0;
  return run_chains(
      host, call, 1, prices_out, ivols_out,
      [&](const auto& g, cudaStream_t s, const cd* phi, cd* lm) {
        launch_hawkes_mgf_sets(s, phi, g.c.P, g.c.M, d_dt.as<double>() + dt0[gi], d_k.as<HawkesMgfConsts>() + g.grid0, g.c.B, g.c.P, lm);
        ++gi;
        return check_launch("hawkes_mgf_sets_kernel");
      },
      d_gam.as<double>(), d_ng.as<double>());
}

/* Hawkes jump-diffusion Fourier chain (hawkesjd_chain_pricer / hawkesjd_chain_pricer_with_risk_premia, hawkes_jd_pricer.py:365-515).
 * risk_premia_gamma = NaN: no risk kernel.  Otherwise the grid sits on Re = -1/2 - gamma, the normalisers / forwards under the risk kernel
 * come from two single-point solves per maturity (each restarted from A = 0) and the gamma slice pricer assembles the prices;
 * normalizers_out / gamma_forwards_out (M each, optional) return them. */
int b200sv_hawkesjd_price_chain(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards, const double* discfactors,
                                const int* offsets, const double* strikes, const int8_t* types, int is_spot_measure, double vol_scaler, int P,
                                double risk_premia_gamma, double* prices_out, double* a_out, double* log_mgf_out, double* normalizers_out,
                                double* gamma_forwards_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out, "null pointer");
  const bool with_gamma = risk_premia_gamma == risk_premia_gamma;
  FourierChain c;
  if (int rc = prepare_hawkes_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure, vol_scaler, P,
                                    risk_premia_gamma))
    return rc;
  P = c.P;
  const HawkesMgfConsts k = make_hawkes_mgf_consts(*params);
  ChainDev d;
  DevBuf d_gam(d.st), d_ng(d.st);
  std::vector<double> ng(2 * (size_t)M, 1.0);                                   // [M][2] (normaliser, gamma forward), 1 without the kernel
  if (with_gamma) {
    if (int rc = risk_kernel_normalizers(d.st, &k, &risk_premia_gamma, 1, M, ttms, forwards, ng)) return rc;
    B200SV_CUDA(d_gam.upload(&risk_premia_gamma, 1));
    B200SV_CUDA(d_ng.upload(ng.data(), ng.size()));
  }
  if (int rc = queue_hawkes_prices(d, c, &k, prices_out, nullptr, d_gam.as<double>(), d_ng.as<double>())) return rc;
  B200SV_CUDA(d.a.download(cplx(a_out), (size_t)M * P * 3));
  B200SV_CUDA(d.lm.download(cplx(log_mgf_out), (size_t)M * P));
  if (int rc = d.sync.done()) return rc;
  for (int m = 0; m < M; ++m) {
    if (normalizers_out) normalizers_out[m] = ng[2 * (size_t)m];
    if (gamma_forwards_out) gamma_forwards_out[m] = ng[2 * (size_t)m + 1];
  }
  return 0;
}

/* Forward-mode sensitivities of the Hawkes Fourier chain without a risk kernel (DESIGN.md §4.3): the pricing launches of
 * b200sv_hawkesjd_price_chain (same function, so bit-identical prices), hawkes_mgf_tangent_kernel, then fourier_vanilla_greeks_kernel on the
 * tangent kernel's own primal log-MGF; one synchronisation at the end. */
int b200sv_hawkesjd_price_chain_greeks(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                       const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                       int is_spot_measure, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                       double* dlog_mgf_out, int* nfev_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && greeks_out, "null pointer");
  FourierChain c;
  if (int rc = prepare_hawkes_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure, vol_scaler, P, NAN))
    return rc;
  const HawkesMgfConsts k = make_hawkes_mgf_consts(*params);
  ChainDev d;
  GreeksDev<kHawkesGreekParams> g(d.st);
  if (int rc = queue_hawkes_greeks(d, g, c, *params, k, prices_out)) return rc;
  return g.download(d, c, greeks_out, dlog_mgf_out, nfev_out);
}

/* Forward-mode sensitivities of the Hawkes Fourier chain under the risk kernel (DESIGN.md §4.12): the launches of
 * queue_hawkes_rp_greeks (bit-identical prices to b200sv_hawkesjd_price_chain with the same gamma); one synchronisation at the end.
 * greeks_out [2 + 16][J]: delta, gamma, HAWKES_GREEK_PARAMS, risk_premia_gamma.  Optional: dlog_mgf_out [16][M][P] (complex),
 * dlog_norm_out [16][M][2] (the derivatives of Re log-MGF at -gamma and -gamma - 1), nfev_out [P]. */
int b200sv_hawkesjd_price_chain_risk_premia_greeks(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                                   const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                                   int is_spot_measure, double vol_scaler, int P, double risk_premia_gamma, double* prices_out,
                                                   double* greeks_out, double* dlog_mgf_out, double* dlog_norm_out, int* nfev_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && greeks_out, "null pointer");
  B200SV_REQUIRE(std::isfinite(risk_premia_gamma), "risk_premia_gamma must be finite");
  FourierChain c;
  if (int rc = prepare_hawkes_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure, vol_scaler, P,
                                    risk_premia_gamma))
    return rc;
  constexpr int NP = kHawkesRpParams;
  const HawkesMgfConsts k = make_hawkes_mgf_consts(*params);
  ChainDev d;
  HawkesRpDev r(d.st);
  GreeksDev<NP> g(d.st);
  if (int rc = queue_hawkes_rp_greeks(d, g, r, c, *params, k, ttms, forwards, risk_premia_gamma, prices_out)) return rc;
  std::vector<cd> dn(dlog_norm_out ? (size_t)NP * M * 2 : 0);
  B200SV_CUDA(r.dn.download(dlog_norm_out ? dn.data() : nullptr, dn.size()));
  if (int rc = g.download(d, c, greeks_out, dlog_mgf_out, nfev_out)) return rc;
  for (size_t i = 0; i < dn.size(); ++i) dlog_norm_out[i] = dn[i].re;
  return 0;
}

/* Second-order sensitivities of the Hawkes Fourier chain under the risk kernel (DESIGN.md §4.13): the launches of
 * b200sv_hawkesjd_price_chain_risk_premia_greeks unchanged (bit-identical first-order outputs), then hawkes_mgf_hessian_kernel<true> on the
 * grid (carried) and at the two normaliser points (restarted), and fourier_gamma_hessian_kernel; one synchronisation at the end. */
int b200sv_hawkesjd_price_chain_risk_premia_hessian(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                                    const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                                    int is_spot_measure, double vol_scaler, int P, double risk_premia_gamma, double* prices_out,
                                                    double* greeks_out, double* dlog_mgf_out, double* dlog_norm_out, int* nfev_out,
                                                    double* vanna_out, double* hessian_out, double* d2log_mgf_out, double* d2log_norm_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && greeks_out && vanna_out && hessian_out, "null pointer");
  B200SV_REQUIRE(std::isfinite(risk_premia_gamma), "risk_premia_gamma must be finite");
  FourierChain c;
  if (int rc = prepare_hawkes_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure, vol_scaler, P,
                                    risk_premia_gamma))
    return rc;
  P = c.P;
  constexpr int NP = kHawkesRpParams, NH = NP * (NP + 1) / 2;
  const HawkesMgfConsts k = make_hawkes_mgf_consts(*params);
  ChainDev d;
  HawkesRpDev r(d.st);
  GreeksDev<NP> g(d.st);
  if (int rc = queue_hawkes_rp_greeks(d, g, r, c, *params, k, ttms, forwards, risk_premia_gamma, prices_out)) return rc;
  const HawkesTangentDirs dirs = make_hawkes_tangents(*params);
  DevBuf d_d2c(d.st), d_d2n(d.st), d_d2lm(d.st), d_v(d.st), d_h(d.st);
  if (int rc = queue_hawkes_hessian<true>(d, c, *params, k, dirs, d_d2c, d_d2lm)) return rc;
  B200SV_CUDA(d_d2n.alloc(sizeof(cd) * (size_t)NH * M * 2));
  if (int rc = launch_hawkes_mgf_hessian<true>(d.st, r.two.as<cd>(), 2, M, r.ttm.as<double>(), k, dirs, d_d2c, 1, d_d2n.as<cd>())) return rc;
  if (c.Jtot > 0) {       // the vanna CTA and NH / NP Hessian CTAs per strike
    B200SV_CUDA(d_v.alloc(sizeof(double) * (size_t)NP * c.Jtot));
    B200SV_CUDA(d_h.alloc(sizeof(double) * (size_t)NH * c.Jtot));
    const dim3 grid(c.Jtot, 1 + (NH + NP - 1) / NP);
    fourier_gamma_hessian_kernel<<<grid, kFourierThreads, 0, d.st>>>(g.lm.as<cd>(), g.dlm.as<cd>(), d_d2lm.as<cd>(), r.dn.as<cd>(),
                                                                     d_d2n.as<cd>(), d.phi.as<cd>(), P, M, d.rows.as<StrikeSpec>(),
                                                                     risk_premia_gamma, r.ng.as<double>(), d_v.as<double>(), d_h.as<double>());
    if (int rc = check_launch("fourier_gamma_hessian_kernel")) return rc;
    B200SV_CUDA(d_v.download(vanna_out, (size_t)NP * c.Jtot));
    B200SV_CUDA(d_h.download(hessian_out, (size_t)NH * c.Jtot));
  }
  B200SV_CUDA(d_d2lm.download(cplx(d2log_mgf_out), (size_t)NH * M * P));
  std::vector<cd> dn(dlog_norm_out ? (size_t)NP * M * 2 : 0), d2n(d2log_norm_out ? (size_t)NH * M * 2 : 0);
  B200SV_CUDA(r.dn.download(dlog_norm_out ? dn.data() : nullptr, dn.size()));
  B200SV_CUDA(d_d2n.download(d2log_norm_out ? d2n.data() : nullptr, d2n.size()));
  if (int rc = g.download(d, c, greeks_out, dlog_mgf_out, nfev_out)) return rc;
  for (size_t i = 0; i < dn.size(); ++i) dlog_norm_out[i] = dn[i].re;
  for (size_t i = 0; i < d2n.size(); ++i) d2log_norm_out[i] = d2n[i].re;
  return 0;
}

/* Second-order sensitivities of the Hawkes Fourier chain without a risk kernel (DESIGN.md §4.5): the launches of
 * b200sv_hawkesjd_price_chain_greeks unchanged (bit-identical first-order outputs), then hawkes_mgf_hessian_kernel<false> and the split
 * second-order sums; one synchronisation at the end. */
int b200sv_hawkesjd_price_chain_hessian(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                        const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                        int is_spot_measure, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                        double* dlog_mgf_out, int* nfev_out, double* vanna_out, double* hessian_out, double* d2log_mgf_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && greeks_out && vanna_out && hessian_out, "null pointer");
  FourierChain c;
  if (int rc = prepare_hawkes_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure, vol_scaler, P, NAN))
    return rc;
  const HawkesMgfConsts k = make_hawkes_mgf_consts(*params);
  ChainDev d;
  GreeksDev<kHawkesGreekParams> g(d.st);
  if (int rc = queue_hawkes_greeks(d, g, c, *params, k, prices_out)) return rc;
  DevBuf d_d2c(d.st), d_d2lm(d.st);
  if (int rc = queue_hawkes_hessian<false>(d, c, *params, k, make_hawkes_tangents(*params), d_d2c, d_d2lm)) return rc;
  // the tangent kernel's primal log-MGF and tangents, as for the first-order rows
  if (int rc = queue_hessian_sums<kHawkesGreekParams>(d, c, g.lm.as<cd>(), g.dlm.as<cd>(), d_d2lm, vanna_out, hessian_out, d2log_mgf_out))
    return rc;
  return g.download(d, c, greeks_out, dlog_mgf_out, nfev_out);
}

/* ---- theta of the three Fourier chain pricers (DESIGN.md §4.8) ----
 * The launches of b200sv_*_price_chain_greeks unchanged (bit-identical outputs), then the theta kernel and fourier_vanilla_greeks_kernel<1>
 * on the log-MGF the parameter rows were summed on; one synchronisation at the end. */
int b200sv_logsv_price_chain_greeks_theta(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                          const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                          const int8_t* types, int is_spot_measure, int variable_type, int expansion_order,
                                          double vol_scaler, int P, double* prices_out, double* greeks_out, double* dlog_mgf_out,
                                          int* nfev_out, double* theta_out, double* dlog_mgf_theta_out, int* theta_nfev_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && greeks_out && theta_out, "null pointer");
  if (variable_type != B200SV_LOG_RETURN) return fail(-4, "variable_type not implemented: sensitivities cover LOG_RETURN only");
  FourierChain c;
  if (int rc = prepare_logsv_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure, variable_type,
                                   expansion_order, vol_scaler, P))
    return rc;
  ChainDev d;
  GreeksDev<1 + kLogsvOdeDirs> g(d.st);
  if (int rc = queue_logsv_greeks(d, g, c, params, etas, expansion_order, prices_out)) return rc;
  ThetaDev t(d.st);
  if (int rc = t.alloc(c, true)) return rc;
  const auto theta = expansion_order == B200SV_ORDER_FIRST ? logsv_mgf_theta_kernel<3> : logsv_mgf_theta_kernel<5>;
  theta<<<(c.P + kThetaTPB - 1) / kThetaTPB, kThetaTPB, 0, d.st>>>(d.phi.as<cd>(), c.P, M, d.spec.as<ChainSpec>(), params->sigma0 - params->theta,
                                                                   t.dlm.as<cd>(), t.nfev.as<int>());
  if (int rc = t.sums(d, c, g.lm.as<cd>())) return rc;
  if (int rc = t.download(c, theta_out, dlog_mgf_theta_out, theta_nfev_out)) return rc;
  if (int rc = g.download(d, c, greeks_out, dlog_mgf_out, nfev_out)) return rc;
  ThetaDev::finish(c, theta_out);
  return 0;
}

int b200sv_heston_price_chain_greeks_theta(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                           const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                           int variable_type, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                           double* dlog_mgf_out, double* theta_out, double* dlog_mgf_theta_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && greeks_out && theta_out, "null pointer");
  if (variable_type != B200SV_LOG_RETURN) return fail(-4, "variable_type not implemented: sensitivities cover LOG_RETURN only");
  FourierChain c;
  if (int rc = prepare_heston_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, variable_type, vol_scaler, P)) return rc;
  ChainDev d;
  GreeksDev<1 + kHestonOdeDirs> g(d.st);
  if (int rc = queue_heston_greeks(d, g, c, params, prices_out)) return rc;
  ThetaDev t(d.st);
  if (int rc = t.alloc(c, false)) return rc;
  heston_mgf_theta_kernel<<<(c.P + 63) / 64, 64, 0, d.st>>>(d.phi.as<cd>(), c.P, M, d.dt.as<double>(), *params, t.dlm.as<cd>());
  if (int rc = t.sums(d, c, d.lm.as<cd>())) return rc;
  if (int rc = t.download(c, theta_out, dlog_mgf_theta_out, nullptr)) return rc;
  if (int rc = g.download(d, c, greeks_out, dlog_mgf_out, nullptr)) return rc;
  ThetaDev::finish(c, theta_out);
  return 0;
}

int b200sv_hawkesjd_price_chain_greeks_theta(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                             const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                             int is_spot_measure, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                             double* dlog_mgf_out, int* nfev_out, double* theta_out, double* dlog_mgf_theta_out,
                                             int* theta_nfev_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && greeks_out && theta_out, "null pointer");
  FourierChain c;
  if (int rc = prepare_hawkes_chain(c, params, M, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure, vol_scaler, P, NAN))
    return rc;
  const HawkesMgfConsts k = make_hawkes_mgf_consts(*params);
  ChainDev d;
  GreeksDev<kHawkesGreekParams> g(d.st);
  if (int rc = queue_hawkes_greeks(d, g, c, *params, k, prices_out)) return rc;
  ThetaDev t(d.st);
  if (int rc = t.alloc(c, true)) return rc;
  hawkes_mgf_theta_kernel<<<(c.P + kThetaTPB - 1) / kThetaTPB, kThetaTPB, 0, d.st>>>(d.phi.as<cd>(), c.P, M, d.dt.as<double>(), k,
                                                                                     t.dlm.as<cd>(), t.nfev.as<int>());
  if (int rc = t.sums(d, c, g.lm.as<cd>())) return rc;
  if (int rc = t.download(c, theta_out, dlog_mgf_theta_out, theta_nfev_out)) return rc;
  if (int rc = g.download(d, c, greeks_out, dlog_mgf_out, nfev_out)) return rc;
  ThetaDev::finish(c, theta_out);
  return 0;
}

/* B Hawkes parameter sets on one chain in one pass (the calibration drivers' objective and its finite-difference neighbours).  The Riccati
 * grids run through the single-set hawkes_mgf_kernel, one launch per set queued back to back: a kernel of its own that read the constants
 * per set from memory contracts its fp64 arithmetic into different fused multiply-adds and moves prices by an ulp (DESIGN.md §9), and the
 * rows must equal b200sv_hawkesjd_price_chain bit for bit.  With gammas, the two restarted single-point solves per (set, maturity) come
 * first and ONE copy back feeds the host-side normalisers / forwards (the same host arithmetic as there).  Then all sets' Fourier sums
 * (vanilla or gamma) in one launch, the Black inversion fused, and one copy back. */
int b200sv_hawkesjd_price_chain_batch(const b200sv_hawkes_params* params, int B, int M, const double* ttms, const double* forwards,
                                      const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                      int is_spot_measure, double vol_scaler, int P, const double* gammas, double* prices_out,
                                      double* ivols_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && strikes && types && prices_out, "null pointer");
  FourierChain c;
  if (int rc = prepare_hawkes_batch(c, params, B, M, ttms, forwards, discfactors, offsets, strikes, types, is_spot_measure, vol_scaler, P,
                                    gammas))
    return rc;
  std::vector<HawkesMgfConsts> k(B);
  for (int b = 0; b < B; ++b) k[b] = make_hawkes_mgf_consts(params[b]);
  ChainDev d;
  DevBuf d_gam(d.st), d_ng(d.st);
  if (gammas) {
    std::vector<double> ng;
    if (int rc = risk_kernel_normalizers(d.st, k.data(), gammas, B, M, ttms, forwards, ng)) return rc;
    B200SV_CUDA(d_ng.upload(ng.data(), ng.size()));
    B200SV_CUDA(d_gam.upload(gammas, (size_t)B));
  }
  if (int rc = queue_hawkes_prices(d, c, k.data(), prices_out, ivols_out, d_gam.as<double>(), d_ng.as<double>())) return rc;
  return d.sync.done();
}


/* compute_hawkes_a_mgf_grid (hawkes_jd_pricer.py:518-547) on caller-supplied grids: A(0) = a_inout [P][3] -> A(dtau) in place, log_mgf_out [P] */
int b200sv_hawkesjd_mgf_grid(const double* phi, const double* psi, int P, double dtau, double* a_inout, const b200sv_hawkes_params* params,
                             double* log_mgf_out) {
  B200SV_REQUIRE(phi && a_inout && params && log_mgf_out, "null pointer");
  B200SV_REQUIRE(P >= 1 && dtau > 0.0, "P >= 1, dtau > 0");
  const HawkesMgfConsts c = make_hawkes_mgf_consts(*params);
  return run_grid(phi, psi, P, a_inout, 3, a_inout, log_mgf_out, [&](cudaStream_t st, const cd* ph, const cd* ps, const cd* a0, cd* a1, cd* lm) {
    DevBuf d_dt(st);
    B200SV_CUDA(d_dt.upload(&dtau, 1));
    launch_hawkes_mgf(st, ph, ps, P, 1, d_dt.as<double>(), c, a0, a1, lm, 0);
    return check_launch("hawkes_mgf_kernel");
  });
}

int b200sv_logsv_mgf_grid(const double* phi, const double* psi, int P, double dtau, double* a_inout,
                          const b200sv_logsv_params* params, double eta, int is_spot_measure, int expansion_order,
                          double* log_mgf_out) {
  B200SV_REQUIRE(phi && a_inout && params && log_mgf_out, "null pointer");
  B200SV_REQUIRE(P >= 1 && dtau > 0.0, "P >= 1, dtau > 0");
  if (int rc = check_expansion_order(expansion_order)) return rc;
  const int N = expansion_order == B200SV_ORDER_FIRST ? 3 : 5;
  const ChainSpec spec{dtau, make_model(*params, eta, is_spot_measure != 0)};
  return run_grid(phi, psi, P, a_inout, N, a_inout, log_mgf_out, [&](cudaStream_t st, const cd* ph, const cd* ps, const cd* a0, cd* a1, cd* lm) {
    DevBuf d_spec(st);
    B200SV_CUDA(d_spec.upload(&spec, 1));
    launch_logsv_mgf(N, st, ph, ps, P, 1, d_spec.as<ChainSpec>(), a0, a1, lm, params->sigma0 - params->theta);
    return check_launch("logsv_mgf_kernel");
  });
}

// func_a_ode_quadratic_terms (pricers/logsv/affine_expansion.py:67-184) for a grid of transform points: the dense tensors the reference
// builds per point -- M [n][n][n] (symmetric in the last two indices), L [n][n], H [n], complex -- written from the SAME row tables
// (make_lane_row / make_coef) the ODE kernels integrate with, and func_rhs (:187-205) evaluated with the production rhs<>() at given A.
// Parity entry points: nothing on the pricing path needs the dense tensors.
int b200sv_logsv_ode_terms(const double* phi, const double* psi, int P, const b200sv_logsv_params* params, double eta, int is_spot_measure,
                           int expansion_order, double* M_out, double* L_out, double* H_out) {
  B200SV_REQUIRE(phi && params && M_out && L_out && H_out, "null pointer");
  B200SV_REQUIRE(P >= 1, "P >= 1");
  if (int rc = check_expansion_order(expansion_order)) return rc;
  const int N = expansion_order == B200SV_ORDER_FIRST ? 3 : 5;
  const LogsvModel model = make_model(*params, eta, is_spot_measure != 0);
  return run_grid(phi, psi, P, nullptr, 0, nullptr, nullptr, [&](cudaStream_t st, const cd* ph, const cd* ps, const cd*, cd*, cd*) {
    const size_t nM = (size_t)P * N * N * N, nL = (size_t)P * N * N, nH = (size_t)P * N;
    DevBuf d_M(st), d_L(st), d_H(st);
    B200SV_CUDA(d_M.alloc(sizeof(cd) * nM));
    B200SV_CUDA(d_L.alloc(sizeof(cd) * nL));
    B200SV_CUDA(d_H.alloc(sizeof(cd) * nH));
    const auto terms = N == 5 ? logsv_ode_terms_kernel<5> : logsv_ode_terms_kernel<3>;
    terms<<<(P + 63) / 64, 64, 0, st>>>(ph, ps, P, model, d_M.as<cd>(), d_L.as<cd>(), d_H.as<cd>());
    if (int rc = check_launch("logsv_ode_terms_kernel")) return rc;
    B200SV_CUDA(d_M.download(cplx(M_out), nM));
    B200SV_CUDA(d_L.download(cplx(L_out), nL));
    B200SV_CUDA(d_H.download(cplx(H_out), nH));
    return 0;
  });
}

int b200sv_logsv_ode_rhs(const double* phi, const double* psi, int P, const double* A, const b200sv_logsv_params* params, double eta,
                         int is_spot_measure, int expansion_order, double* rhs_out) {
  B200SV_REQUIRE(phi && A && params && rhs_out, "null pointer");
  B200SV_REQUIRE(P >= 1, "P >= 1");
  if (int rc = check_expansion_order(expansion_order)) return rc;
  const int N = expansion_order == B200SV_ORDER_FIRST ? 3 : 5;
  const LogsvModel model = make_model(*params, eta, is_spot_measure != 0);
  return run_grid(phi, psi, P, A, N, rhs_out, nullptr, [&](cudaStream_t st, const cd* ph, const cd* ps, const cd* a, cd* r, cd*) {
    const auto rhs = N == 5 ? logsv_ode_rhs_kernel<5> : logsv_ode_rhs_kernel<3>;
    rhs<<<(P + 63) / 64, 64, 0, st>>>(ph, ps, P, model, a, r);
    return check_launch("logsv_ode_rhs_kernel");
  });
}

int b200sv_ode_rhs_dense(const double* A, int P, int n, const double* M, const double* L, const double* H, double* rhs_out) {
  B200SV_REQUIRE(A && M && L && H && rhs_out, "null pointer");
  B200SV_REQUIRE(P >= 1 && n >= 1 && n <= 16, "P >= 1, 1 <= n <= 16");
  HostCall call;
  const cudaStream_t st = call.st;
  DevBuf d_A(st), d_M(st), d_L(st), d_H(st), d_R(st);
  B200SV_CUDA(d_A.upload(cplx(A), (size_t)P * n));
  B200SV_CUDA(d_M.upload(cplx(M), (size_t)n * n * n));
  B200SV_CUDA(d_L.upload(cplx(L), (size_t)n * n));
  B200SV_CUDA(d_H.upload(cplx(H), n));
  B200SV_CUDA(d_R.alloc(sizeof(cd) * (size_t)P * n));
  ode_rhs_dense_kernel<<<(P * n + 127) / 128, 128, 0, st>>>(d_A.as<cd>(), P, n, d_M.as<cd>(), d_L.as<cd>(), d_H.as<cd>(), d_R.as<cd>());
  if (int rc = check_launch("ode_rhs_dense_kernel")) return rc;
  B200SV_CUDA(d_R.download(cplx(rhs_out), (size_t)P * n));
  return call.sync.done();
}

// compute_logsv_a_mgf_grid(is_analytic=True): the semi-analytic branch over a transform grid (affine_expansion.py:388-470 -> :306-384)
int b200sv_logsv_mgf_grid_analytic(const double* phi, const double* psi, int P, double dtau, double* a_inout, const b200sv_logsv_params* params,
                                   int is_spot_measure, int expansion_order, int year_days, double* log_mgf_out) {
  B200SV_REQUIRE(phi && a_inout && params && log_mgf_out, "null pointer");
  B200SV_REQUIRE(P >= 1 && dtau > 0.0 && year_days >= 1, "P >= 1, dtau > 0, year_days >= 1");
  if (int rc = check_expansion_order(expansion_order)) return rc;
  const int N = expansion_order == B200SV_ORDER_FIRST ? 3 : 5;
  const LogsvModel model = make_model(*params, 1.0, is_spot_measure != 0);      // eta is ignored on this branch (reference :340-348)
  return run_grid(phi, psi, P, a_inout, N, a_inout, log_mgf_out, [&](cudaStream_t st, const cd* ph, const cd* ps, const cd* a0, cd* a1, cd* lm) {
    const auto analytic = N == 5 ? logsv_mgf_analytic_kernel<5> : logsv_mgf_analytic_kernel<3>;
    analytic<<<(P + 63) / 64, 64, 0, st>>>(ph, ps, P, model, dtau, year_days, a0, a1, lm, params->sigma0 - params->theta);
    return check_launch("logsv_mgf_analytic_kernel");
  });
}

// compute_logsv_a_mgf_grid(is_stiff_solver=True): SciPy's BDF control law per grid point (affine_expansion.py:229-303)
int b200sv_logsv_mgf_grid_bdf(const double* phi, const double* psi, int P, double dtau, double* a_inout, const b200sv_logsv_params* params,
                              double eta, int is_spot_measure, int expansion_order, double* log_mgf_out) {
  B200SV_REQUIRE(phi && a_inout && params && log_mgf_out, "null pointer");
  B200SV_REQUIRE(P >= 1 && dtau > 0.0, "P >= 1, dtau > 0");
  if (int rc = check_expansion_order(expansion_order)) return rc;
  const int N = expansion_order == B200SV_ORDER_FIRST ? 3 : 5;
  const LogsvModel model = make_model(*params, eta, is_spot_measure != 0);
  return run_grid(phi, psi, P, a_inout, N, a_inout, log_mgf_out, [&](cudaStream_t st, const cd* ph, const cd* ps, const cd* a0, cd* a1, cd* lm) {
    const auto bdf = N == 5 ? logsv_mgf_bdf_kernel<5> : logsv_mgf_bdf_kernel<3>;
    bdf<<<(P + 63) / 64, 64, 0, st>>>(ph, ps, P, model, dtau, a0, a1, lm, params->sigma0 - params->theta, nullptr);
    return check_launch("logsv_mgf_bdf_kernel");
  });
}

int b200sv_heston_mgf_grid(const double* phi, const double* psi, int P, double dtau, double* a_inout, double* b_inout,
                           const b200sv_heston_params* params, double* log_mgf_out) {
  B200SV_REQUIRE(phi && a_inout && b_inout && params && log_mgf_out, "null pointer");
  B200SV_REQUIRE(P >= 1 && dtau > 0.0, "P >= 1, dtau > 0");
  return run_grid(phi, psi, P, a_inout, 1, a_inout, log_mgf_out, [&](cudaStream_t st, const cd* ph, const cd* ps, const cd* a0, cd* a1, cd* lm) {
    DevBuf d_dt(st), d_b(st), d_b1(st);
    B200SV_CUDA(d_dt.upload(&dtau, 1));
    B200SV_CUDA(d_b.upload(cplx(b_inout), P));
    B200SV_CUDA(d_b1.alloc(sizeof(cd) * P));
    const int tpb = mgf_block_threads(P);
    heston_mgf_kernel<<<(P + tpb - 1) / tpb, tpb, 0, st>>>(ph, ps, P, 1, d_dt.as<double>(), *params, a0, d_b.as<cd>(), a1, d_b1.as<cd>(), lm,
                                                           nullptr, 0);
    if (int rc = check_launch("heston_mgf_kernel")) return rc;
    B200SV_CUDA(d_b1.download(cplx(b_inout), P));
    return 0;
  });
}

int b200sv_fourier_vanilla(const double* log_mgf, const double* phi, int P, double forward, const double* strikes,
                           const int8_t* types, int J, double discfactor, int is_spot_measure, double* prices_out) {
  B200SV_REQUIRE(log_mgf && phi && strikes && types && prices_out, "null pointer");
  B200SV_REQUIRE(P >= 3 && J >= 1, "P >= 3, J >= 1");
  const bool spot = is_spot_measure != 0;
  if (int rc = check_fourier_types(types, J, spot)) return rc;
  std::vector<StrikeSpec> ss(J);
  for (int j = 0; j < J; ++j) ss[j] = StrikeSpec{strikes[j], forward, discfactor, (int)types[j], 0, 1.0, 0};
  const int half_re = all_half_re(phi, P) ? 1 : 0;
  return run_sums(log_mgf, phi, P, ss, prices_out, [&](cudaStream_t st, unsigned n, const cd* lm, const cd* g, const StrikeSpec* s, double* pr) {
    fourier_vanilla_kernel<<<n, kFourierThreads, 0, st>>>(lm, g, P, s, spot ? 1 : 0, half_re, pr, nullptr);
    return check_launch("fourier_vanilla_kernel");
  });
}

/* slice_pricer_with_mgf_grid_with_gamma (utils/mgf_pricer.py:273-320) on caller-supplied log-MGF / transform grids: 'C' / 'P' under the spot
 * measure, everything else is ValueError("not implemented") there (-5 here) */
int b200sv_fourier_gamma(const double* log_mgf, const double* phi, int P, double risk_premia_gamma, double forward, double normalizer,
                         double gamma_forward, const double* strikes, const int8_t* types, int J, int is_spot_measure, double* prices_out) {
  B200SV_REQUIRE(log_mgf && phi && strikes && types && prices_out, "null pointer");
  B200SV_REQUIRE(P >= 3 && J >= 1, "P >= 3, J >= 1");
  if (int rc = check_gamma_types(types, J, is_spot_measure != 0)) return rc;
  std::vector<StrikeSpec> ss(J);
  for (int j = 0; j < J; ++j) ss[j] = StrikeSpec{strikes[j], forward, 1.0, (int)types[j], 0, 1.0, 0};
  const double ng[2] = {normalizer, gamma_forward};
  return run_sums(log_mgf, phi, P, ss, prices_out, [&](cudaStream_t st, unsigned n, const cd* lm, const cd* g, const StrikeSpec* s, double* pr) {
    DevBuf d_gam(st), d_ng(st);
    B200SV_CUDA(d_gam.upload(&risk_premia_gamma, 1));
    B200SV_CUDA(d_ng.upload(ng, 2));
    fourier_gamma_batch_kernel<<<n, kFourierThreads, 0, st>>>(lm, g, P, s, d_gam.as<double>(), d_ng.as<double>(), pr, nullptr);
    return check_launch("fourier_gamma_batch_kernel");
  });
}

int b200sv_fourier_qvar(const double* log_mgf, const double* psi, int P, double ttm, const double* strikes, const int8_t* types, int J,
                        double discfactor, double* prices_out) {
  B200SV_REQUIRE(log_mgf && psi && strikes && types && prices_out, "null pointer");
  B200SV_REQUIRE(P >= 3 && J >= 1 && ttm > 0.0, "P >= 3, J >= 1, ttm > 0");
  if (int rc = check_qvar_types(types, J)) return rc;
  std::vector<SumSpec> specs(J);
  for (int j = 0; j < J; ++j) specs[j] = SumSpec{strikes[j] * ttm, discfactor, ttm, (int)types[j], 0};
  return fourier_sum_host(log_mgf, psi, P, specs, kModeQvar, 0, prices_out);
}

int b200sv_fourier_pdf(const double* log_mgf, const double* grid, int P, const double* z, int J, double* out) {
  B200SV_REQUIRE(log_mgf && grid && z && out, "null pointer");
  B200SV_REQUIRE(P >= 3 && J >= 1, "P >= 3, J >= 1");
  std::vector<SumSpec> specs(J);
  for (int j = 0; j < J; ++j) specs[j] = SumSpec{z[j], 1.0, 1.0, 0, 0};
  return fourier_sum_host(log_mgf, grid, P, specs, kModePdf, 0, out);
}

int b200sv_fourier_digital(const double* log_mgf, const double* phi, int P, double forward, const double* strikes, const int8_t* types,
                           int J, double discfactor, double* prices_out) {
  B200SV_REQUIRE(log_mgf && phi && strikes && types && prices_out, "null pointer");
  B200SV_REQUIRE(P >= 3 && J >= 1, "P >= 3, J >= 1");
  for (int j = 0; j < J; ++j)
    if (types[j] != B200SV_CALL && types[j] != B200SV_PUT) return fail(-5, "not implemented");   // utils/mgf_pricer.py:265-266
  bool all_neg = true;                                             // np.all(np.real(phi_grid) < 0.0), :241
  for (int i = 0; i < P; ++i) all_neg = all_neg && (phi[2 * i] < 0.0);
  std::vector<SumSpec> specs(J);
  for (int j = 0; j < J; ++j) specs[j] = SumSpec{-std::log(forward / strikes[j]), discfactor, 1.0, (int)types[j], 0};
  return fourier_sum_host(log_mgf, phi, P, specs, kModeDigital, all_neg ? 1 : 0, prices_out);
}

}  // extern "C"
