// mc_kernels.cu -- fused Monte Carlo hot path for sm_90a (H100).
//
// Replaces, behind the C ABI of include/b200sv.h, the reference functions (paths under
// /root/reference/src/stochvolmodels):
//   simulate_logsv_x_vol_terminal     pricers/logsv_pricer.py:950-1047
//   logsv_mc_chain_pricer             pricers/logsv_pricer.py:806-867
//   logsv_mc_chain_pricer_fixed_randoms (stepping part)  pricers/logsv_pricer.py:1100-1162
//   simulate_heston_x_vol_terminal    pricers/heston_pricer.py:334-381
//   heston_mc_chain_pricer            pricers/heston_pricer.py:285-331
//   compute_mc_vars_payoff            utils/mc_payoffs.py:10-88
//   set_time_grid                     utils/funcs.py:24-47
//
// Design (DESIGN.md §3): one persistent wave of CTAs; a thread owns one path at a time, keeps (x, log sigma, sigma,
// sigma^2, qvar) in registers for the whole maturity slice, draws its Gaussians in-kernel (Philox4x32-10 keyed by the
// GLOBAL path id), and touches HBM only to load / store the SoA state at slice boundaries (24 B + 24 B per path per slice
// in fp64).  The forward re-centring of the payoffs needs the mean over ALL paths first, hence two phases per slice:
//   slice kernel  -> per-CTA (sum F e^x, count) partials -> fixed-order reduction            [all-reduce #1 if multi-GPU]
//   payoff kernel -> per-CTA per-strike (sum, sum^2, count) partials -> fixed-order reduction [all-reduce #2 if multi-GPU]
// All moment arithmetic is fp64 and every reduction has a fixed order => bitwise reproducible for a given launch shape.
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>
#include <type_traits>
#include <cstdlib>
#include <vector>

#include "../../include/b200sv.h"
#include "common.cuh"
#include "fastmath64.cuh"
#include "p2p.cuh"
#include "black.cuh"
#include "philox.cuh"

namespace b200sv {

cudaStream_t& current_stream_ref() {
  static thread_local cudaStream_t st = nullptr;
  return st;
}
long long& launch_count_ref() {
  static thread_local long long n = 0;
  return n;
}
constexpr int kThreads = 256;
#ifndef B200SV_SLICE_PREFETCH
#define B200SV_SLICE_PREFETCH 1     // issue the next Philox/Box-Muller call before the two fp64 steps of the current one
#endif
#ifndef B200SV_SLICE_THREADS
#define B200SV_SLICE_THREADS 256
#endif
constexpr int kSliceThreads = B200SV_SLICE_THREADS;
#ifndef B200SV_SLICE_MINBLOCKS
#define B200SV_SLICE_MINBLOCKS 2   // resident CTAs / SM the slice kernel is register-budgeted for: 2 x 256 threads = 16 warps/SM at <= 128
#endif                             // registers/thread of the 64K-entry register file (tools/occupancy_sweep.sh sweeps the alternatives)
constexpr int kStrikeChunk = 8;

// --------------------------------------------------------------------------------------------------------------------
// per-step model updates
// --------------------------------------------------------------------------------------------------------------------
struct LogsvConsts {   // all dt / sqrt(dt) factors folded in on the host (fp64)
  double cx;    // alpha * 0.5 * eta^2 * dt          x  += cx * sigma^2 + ce * sigma * z0
  double ce;    // eta * sqrt(dt)
  double a0;    // (-kappa1 + kappa2*theta - 0.5*vartheta^2) * dt
  double a1;    // kappa1 * theta * dt               L  += a0 + a1 / sigma + a2 * sigma + b0 z0 + b1 z1
  double a2;    // (adj - kappa2) * dt
  double b0;    // beta * sqrt(dt)
  double b1;    // volvol * sqrt(dt)
  double cq;    // 0.5 * eta^2 * dt                  q  += cq * (sigma_old^2 + sigma_new^2)
  double a0s, a1s, a2s, b0s, b1s;   // a0..b1 in table units (x 256/ln2): the fp64 stepper carries Ls = L * 256/ln2 (fastmath64.cuh)
};

struct HestonConsts {
  double hx;    // -0.5 * dt                         x += hx * v + sdt * sqrt(v) * z0
  double sdt;   // sqrt(dt)
  double dt;    //                                   q += dt * v
  double kdt;   // kappa * dt                        v += kdt * (theta - v) + sqrt(v) * (c0 z0 + c1 z1);  v = max(v, 1e-4)
  double theta;
  double c0;    // volvol * rho * sqrt(dt)
  double c1;    // volvol * sqrt(1 - rho^2) * sqrt(dt)
  // opt-in Andersen (2008) quadratic-exponential scheme (B200SV_HESTON_QE), central discretisation gamma1 = gamma2 = 1/2
  int qe;
  double e;     // exp(-kappa dt)                     m  = v e + m0,  m0 = theta (1 - e)
  double m0;
  double s1;    // volvol^2 e (1 - e) / kappa         s2 = v s1 + s0
  double s0;    // theta volvol^2 (1 - e)^2 / (2 kappa)
  double K0, K1, K2, K3, K4;   // x' = x + K0 + K1 v + K2 v' + sqrt(K3 v + K4 v') Zx
};

static LogsvConsts make_logsv_consts(const b200sv_logsv_params& p, double eta, bool spot, double dt) {
  // measure switch: pricers/logsv_pricer.py:1032-1035
  const double alpha = spot ? -1.0 : 1.0, adj = spot ? 0.0 : p.beta * eta;
  const double vt2 = p.beta * p.beta + p.volvol * p.volvol, sdt = std::sqrt(dt);
  LogsvConsts c;
  c.cx = alpha * 0.5 * eta * eta * dt;
  c.ce = eta * sdt;
  c.a0 = (-p.kappa1 + p.kappa2 * p.theta - 0.5 * vt2) * dt;
  c.a1 = p.kappa1 * p.theta * dt;
  c.a2 = (adj - p.kappa2) * dt;
  c.b0 = p.beta * sdt;
  c.b1 = p.volvol * sdt;
  c.cq = 0.5 * eta * eta * dt;
  c.a0s = c.a0 * kLogScale;
  c.a1s = c.a1 * kLogScale;
  c.a2s = c.a2 * kLogScale;
  c.b0s = c.b0 * kLogScale;
  c.b1s = c.b1 * kLogScale;
  return c;
}

static HestonConsts make_heston_consts(const b200sv_heston_params& p, double dt, int scheme = B200SV_HESTON_EULER_FLOOR) {
  const double sdt = std::sqrt(dt);
  HestonConsts c;
  c.qe = scheme == B200SV_HESTON_QE;
  c.e = std::exp(-p.kappa * dt);
  c.m0 = p.theta * (1.0 - c.e);
  c.s1 = p.volvol * p.volvol * c.e * (1.0 - c.e) / p.kappa;
  c.s0 = p.theta * p.volvol * p.volvol * (1.0 - c.e) * (1.0 - c.e) / (2.0 * p.kappa);
  const double kre = p.kappa * p.rho / p.volvol;
  c.K0 = -p.rho * p.kappa * p.theta * dt / p.volvol;
  c.K1 = 0.5 * dt * (kre - 0.5) - p.rho / p.volvol;
  c.K2 = 0.5 * dt * (kre - 0.5) + p.rho / p.volvol;
  c.K3 = 0.5 * dt * (1.0 - p.rho * p.rho);
  c.K4 = c.K3;
  c.hx = -0.5 * dt;
  c.sdt = sdt;
  c.dt = dt;
  c.kdt = p.kappa * dt;
  c.theta = p.theta;
  c.c0 = p.volvol * p.rho * sdt;
  c.c1 = p.volvol * std::sqrt(1.0 - p.rho * p.rho) * sdt;
  return c;
}

template <typename Real>
struct LogsvPath;

// fp64 state: same scheme, reformulated so that the per-step work is the log-vol recursion plus two running sums:
//   A  = sum_{k=1..S} sigma_k^2      (new sigma of every step)
//   XM = sum_{k=0..S-1} sigma_k z0_k (martingale part of x, old sigma)
// from which  x_S = x_0 + cx*(sigma_0^2 + A - sigma_S^2) + ce*XM          [sum_k cx*sigma_k^2 + ce*sigma_k*z0_k]
//             q_S = q_0 + cq*(sigma_0^2 + 2A - sigma_S^2)                 [sum_k cq*(sigma_k^2 + sigma_{k+1}^2)]
// (logsv_pricer.py:1041-1045 summed over the slice).  The log-vol is carried in table units Ls = L * 256/ln2 so that sigma = exp(L) and
// 1/sigma = exp(-L) come out of exp_pair_scaled (11 fp64 instructions, fastmath64.cuh); 18 fp64-pipe instructions per step in all.
// Range guard: step<false> only RECORDS |Ls| > kLogScaledMax (|L| > 699.997: one LOP3 + one ISETP.OR per step); a path that ever trips
// it is re-run by the kernel with step<true>, which clamps every step -- the result is the clamped recursion for every path, the common
// case pays 2 integer instructions instead of 5 + 2.
template <>
struct LogsvPath<double> {
  double Ls, s, inv, A, XM, x0, q0, s2_first;
  double cx, ce, a0, a1, a2, b0, b1, cq;
  bool bad;
  __device__ __forceinline__ LogsvPath(const LogsvConsts& c)
      : cx(c.cx), ce(c.ce), a0(c.a0s), a1(c.a1s), a2(c.a2s), b0(c.b0s), b1(c.b1s), cq(c.cq), bad(false) {}
  __device__ __forceinline__ void load(double x_, double sigma0, double q_) {
    x0 = x_;
    q0 = q_;
    Ls = clamp_log_scaled(clamp_log(log(sigma0)) * kLogScale);    // vol_var = np.log(sigma0), logsv_pricer.py:1039
    exp_pair_scaled(Ls, s, inv);
    s = sigma0;                    // keep the loaded sigma itself for the first step
    s2_first = s * s;
    A = 0.0;
    XM = 0.0;
    bad = false;
  }
  template <bool SAFE>
  __device__ __forceinline__ void step(double z0, double z1) {
#if defined(B200SV_ABLATE) && (B200SV_ABLATE & 4)   // tuning only: no fp64 recursion, just consume the normals
    XM = fma(z1, z0, XM);
    return;
#endif
    XM = fma(s, z0, XM);
    // noise + constant drift first (independent of sigma: off the critical path), then the two state-dependent terms
    double l = Ls + fma(b0, z0, fma(b1, z1, a0));
    l = fma(a2, s, l);
    l = fma(a1, inv, l);
    if constexpr (SAFE)
      l = clamp_log_scaled(l);
    else
      bad |= log_scaled_out_of_range(l);
    Ls = l;
    exp_pair_scaled(Ls, s, inv);
    A = fma(s, s, A);
  }
  __device__ __forceinline__ bool overflowed() const { return bad; }
  __device__ __forceinline__ double sigma() const { return s; }
  __device__ __forceinline__ double x() const { return fma(ce, XM, fma(cx, (s2_first - s * s) + A, x0)); }
  __device__ __forceinline__ double q() const { return fma(cq, (s2_first - s * s) + 2.0 * A, q0); }
};

// fp32 state (opt-in B200SV_STATE_F32): same structure, SFU exp / reciprocal
template <>
struct LogsvPath<float> {
  float L, s, inv, A, XM, x0, q0, s2_first;
  float cx, ce, a0, a1, a2, b0, b1, cq;
  __device__ __forceinline__ LogsvPath(const LogsvConsts& c)
      : cx((float)c.cx), ce((float)c.ce), a0((float)c.a0), a1((float)c.a1), a2((float)c.a2), b0((float)c.b0),
        b1((float)c.b1), cq((float)c.cq) {}
  __device__ __forceinline__ void load(float x_, float sigma0, float q_) {
    x0 = x_;
    q0 = q_;
    L = __logf(sigma0);
    s = sigma0;
    s2_first = s * s;
    inv = __frcp_rn(s);
    A = 0.0f;
    XM = 0.0f;
  }
  template <bool SAFE>
  __device__ __forceinline__ void step(float z0, float z1) {
    XM = fmaf(s, z0, XM);
    float l = L + fmaf(b0, z0, fmaf(b1, z1, a0));
    l = fmaf(a2, s, l);
    l = fmaf(a1, inv, l);
    L = fminf(fmaxf(l, -80.0f), 80.0f);
    s = __expf(L);
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"(s));
    A = fmaf(s, s, A);
  }
  __device__ __forceinline__ bool overflowed() const { return false; }   // L is clamped every step
  __device__ __forceinline__ float sigma() const { return s; }
  __device__ __forceinline__ float x() const { return fmaf(ce, XM, fmaf(cx, (s2_first - s * s) + A, x0)); }
  __device__ __forceinline__ float q() const { return fmaf(cq, (s2_first - s * s) + 2.0f * A, q0); }
};

// QE = compile-time scheme switch: the floor-Euler kernel carries none of the quadratic-exponential code (a runtime flag inside the step
// cost the reference scheme 6 % through registers and instruction-cache footprint)
template <typename Real, bool QE = false>
struct HestonPath {
  Real v, V, XM, x0, q0, xacc, qacc;
  Real hx, sdt, dt, kdt, theta, c0, c1;
  Real e, m0, s1, s0, K0, K1, K2, K3, K4;
  int qe;
  __device__ __forceinline__ HestonPath(const HestonConsts& c)
      : hx((Real)c.hx), sdt((Real)c.sdt), dt((Real)c.dt), kdt((Real)c.kdt), theta((Real)c.theta), c0((Real)c.c0), c1((Real)c.c1),
        e((Real)c.e), m0((Real)c.m0), s1((Real)c.s1), s0((Real)c.s0), K0((Real)c.K0), K1((Real)c.K1), K2((Real)c.K2), K3((Real)c.K3),
        K4((Real)c.K4), qe(c.qe) {}
  __device__ __forceinline__ void load(Real x_, Real v_, Real q_) {
    x0 = x_;
    v = v_;
    q0 = q_;
    V = (Real)0;
    XM = (Real)0;
    xacc = (Real)0;
    qacc = (Real)0;
  }
  // Andersen's QE step: moment-matched quadratic (psi <= 1.5) or exponential (psi > 1.5) variance draw, then the log-spot with the
  // central discretisation.  z0 drives the spot, z1 the variance (U = Phi(z1) in the exponential branch).  Not in the reference
  // (BASELINE.json names it; SURVEY.md §0.1): validated against the Heston Fourier price and the oracle restatement.
  __device__ __forceinline__ void step_qe(Real zx, Real zv) {
    const Real m = fma(v, e, m0);
    const Real s2 = fma(v, s1, s0);
    const Real mm = m * m;
    Real vn;
    if (s2 <= (Real)1.5 * mm) {          // psi = s2 / m^2 <= 1.5, tested without the division
      // 2/psi = 2 m^2 / s2;  b^2 = 2/psi - 1 + sqrt(2/psi) sqrt(2/psi - 1) with the two roots merged (2/psi >= 4/3: both factors positive);
      // fp64 divisions and square roots through MUFU seeds + Newton / Householder steps (fastmath64.cuh, gauss64.cuh): <= 2 ulp, a third of
      // the instructions of the IEEE routines -- the QE step is 3 divisions + 4 roots in its textbook form, 2 + 3 here
      const Real ip = (Real)2 * fast_div(mm, s2);
      const Real t = ip - (Real)1;
      const Real b2 = t + fast_sqrt(ip * t);
      const Real a = fast_div(m, (Real)1 + b2);
      const Real r = fast_sqrt(b2) + zv;
      vn = a * r * r;
    } else {
      const Real psi = s2 / mm;
      const Real p = (psi - (Real)1) / (psi + (Real)1);
      const Real beta = ((Real)1 - p) / m;
      const Real u = (Real)normcdf((double)zv);
      vn = u <= p ? (Real)0 : (Real)log((double)(((Real)1 - p) / ((Real)1 - u))) / beta;
    }
    const Real arg = K3 * v + K4 * vn;
    xacc += K0 + K1 * v + K2 * vn + (arg > (Real)0 ? fast_sqrt(arg) : (Real)0) * zx;
    qacc += (Real)0.5 * dt * (v + vn);
    v = vn;
  }
  // pricers/heston_pricer.py:372-379 (floor-Euler): everything on the OLD variance, then v = max(v, 1e-4).
  // V = sum v_k, XM = sum sqrt(v_k) z0_k  =>  x_S = x_0 - 0.5*dt*V + sqrt(dt)*XM,  q_S = q_0 + dt*V.
  template <bool SAFE>
  __device__ __forceinline__ void step(Real z0, Real z1) {
    if constexpr (QE) {
      step_qe(z0, z1);
      return;
    }
    const Real sig = sqrt(v);
    V += v;
    XM = fma(sig, z0, XM);
    Real vn = fma(kdt, theta - v, v);
    vn = fma(sig, fma(c0, z0, c1 * z1), vn);
    v = vn > (Real)1e-4 ? vn : (Real)1e-4;     // np.maximum(var0, 1e-4)
  }
  __device__ __forceinline__ bool overflowed() const { return false; }
  __device__ __forceinline__ Real sigma() const { return v; }
  __device__ __forceinline__ Real x() const { return fma(sdt, XM, fma(hx, V, x0)) + xacc; }
  __device__ __forceinline__ Real q() const { return fma(dt, V, q0) + qacc; }
};

// --------------------------------------------------------------------------------------------------------------------
// fused slice kernel
// --------------------------------------------------------------------------------------------------------------------
template <typename Real>
struct SliceArgs {
  Real* x;
  Real* v;      // sigma (LogSV) or variance (Heston)
  Real* q;
  long long n;
  unsigned long long path_offset;
  int init;
  double v_init;
  int nsteps;
  unsigned int slice;
  unsigned long long seed;
  double forward;
  double* partials;   // [gridDim.x][K] re-centring moments (SpotMoments)
};

// advance one path through the slice, drawing its normals in the order philox.cuh defines.  SAFE = clamp the log-vol every step (re-run
// of a path whose fast pass left the representable range); !SAFE = the production loop with the generator software-pipelined one call
// ahead of the fp64 recursion (the integer / SFU stream of call c+1 overlaps the fp64 stream of call c inside a warp).
// PREFETCH = false: no software pipelining (register-bound callers).
template <bool SAFE, bool PREFETCH = (B200SV_SLICE_PREFETCH != 0), typename Path, typename Real, int GAUSS>
__device__ __forceinline__ void run_slice_steps(Path& p, StepNormals<Real, GAUSS>& rng, int nsteps) {
  if constexpr (GAUSS == kGaussF64) {
    if constexpr (SAFE || !PREFETCH) {
      for (int s = 0; s < nsteps; ++s) {
        Real z0, z1;
        rng.get((uint32_t)s, z0, z1);
        p.template step<SAFE>(z0, z1);
      }
    } else {
      Real n0, n1;
      rng.get(0u, n0, n1);
#pragma unroll 1
      for (int s = 0; s < nsteps; ++s) {
        Real m0, m1;
        rng.get((uint32_t)(s + 1), m0, m1);
        p.template step<SAFE>(n0, n1);
        n0 = m0;
        n1 = m1;
      }
    }
  } else {
    // one Philox call feeds two steps
    const int ncalls = nsteps >> 1;
    if constexpr (SAFE || !PREFETCH) {
      for (int c = 0; c < ncalls; ++c) {
        Real n0, n1, n2, n3;
        rng.get2((uint32_t)c, n0, n1, n2, n3);
        p.template step<SAFE>(n0, n1);
        p.template step<SAFE>(n2, n3);
      }
      if (nsteps & 1) {
        Real n0, n1, n2, n3;
        rng.get2((uint32_t)ncalls, n0, n1, n2, n3);
        p.template step<SAFE>(n0, n1);
      }
    } else {
      Real n0, n1, n2, n3, m0, m1, m2, m3;
      rng.get2(0u, n0, n1, n2, n3);
      int c = 0;
#pragma unroll 1
      for (; c + 2 <= ncalls; c += 2) {     // two calls = four steps per iteration: the n / m register sets swap roles, no moves
        rng.get2((uint32_t)(c + 1), m0, m1, m2, m3);
        p.template step<SAFE>(n0, n1);
        p.template step<SAFE>(n2, n3);
        rng.get2((uint32_t)(c + 2), n0, n1, n2, n3);
        p.template step<SAFE>(m0, m1);
        p.template step<SAFE>(m2, m3);
      }
      if (c < ncalls) {
        rng.get2((uint32_t)(c + 1), m0, m1, m2, m3);
        p.template step<SAFE>(n0, n1);
        p.template step<SAFE>(n2, n3);
        n0 = m0;
        n1 = m1;
      }
      if (nsteps & 1) p.template step<SAFE>(n0, n1);
    }
  }
}

// The re-centring moments of one CTA, row blockIdx.x of the partials [gridDim.x][K] that reduce_partials_kernel sums: (sum F e^x, count)
// over the non-NaN spots (spots_t = forward*np.exp(x0), nanmean over all paths, utils/mc_payoffs.py:61-62) and, for K > 2, the K - 2
// tangent terms sum F e^x d_k over the same spots.
template <int K, int THREADS>
struct SpotMoments {
  double acc[K];
  __device__ __forceinline__ SpotMoments() {
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k] = 0.0;
  }
  __device__ __forceinline__ void add(double spot) {
    if (spot == spot) {
      acc[0] += spot;
      acc[1] += 1.0;
    }
  }
  // tangent term k, d = the path's k-th log-spot tangent.  A separate call per k: each kernel keeps its own order of the term and base
  // updates (and of its tangent stores), which its SASS follows.
  __device__ __forceinline__ void add_term(double spot, int k, double d) {
    if (spot == spot) acc[2 + k] = fma(spot, d, acc[2 + k]);
  }
  // block reduction, then thread 0 writes the CTA's row
  __device__ __forceinline__ void store(double* __restrict__ partials) {
    __shared__ double red[K * THREADS / 32];
    block_sum<K, THREADS>(acc, red);
    if (threadIdx.x == 0) {
#pragma unroll
      for (int k = 0; k < K; ++k) partials[K * blockIdx.x + k] = acc[k];
    }
  }
};

// One path of one slice: load the state (or start it from (0, v_init, 0)), step it, re-run it with the per-step clamp if the fast pass
// left the representable log-vol range (rare: |log sigma| > 700 somewhere on the path), store it; returns the terminal x.
template <typename Path, typename Real, int GAUSS>
__device__ __forceinline__ Real slice_path(Path& p, const SliceArgs<Real>& a, long long i) {
  Real xi = (Real)0, vi = (Real)a.v_init, qi = (Real)0;
  if (!a.init) {
    xi = a.x[i];
    vi = a.v[i];
    qi = a.q[i];
  }
  p.load(xi, vi, qi);
  StepNormals<Real, GAUSS> rng(a.seed, a.path_offset + (unsigned long long)i, a.slice);
  run_slice_steps<false>(p, rng, a.nsteps);
  if (p.overflowed()) {
    p.load(xi, vi, qi);
    run_slice_steps<true>(p, rng, a.nsteps);
  }
  const Real xT = p.x();
  a.x[i] = xT;
  a.v[i] = p.sigma();
  a.q[i] = p.q();
  return xT;
}

template <typename Path, typename Consts, typename Real, int GAUSS>
__global__ void __launch_bounds__(kSliceThreads, B200SV_SLICE_MINBLOCKS) mc_slice_kernel(SliceArgs<Real> a, Consts consts) {
  exp_table_init();
  if constexpr (GAUSS != kGaussF32) gauss64_table_init();
  SpotMoments<2, kSliceThreads> mom;
  Path p(consts);
  const long long stride = (long long)gridDim.x * kSliceThreads;
  for (long long i = (long long)blockIdx.x * kSliceThreads + threadIdx.x; i < a.n; i += stride)
    mom.add(a.forward * exp((double)slice_path<Path, Real, GAUSS>(p, a, i)));
  mom.store(a.partials);
}

// out[k] = sum_b partials[b*K + k] for k < K_out, fixed order: one warp per k, lanes stride over b, shuffle tree.
// With a P2P context the same kernel PUBLISHES the K_out values into every peer's mailbox (stores to NVLink-mapped peer memory)
// and then signals the epoch -- the producer half of the exchange, fused into the reduction that produces the values (p2p.cuh).
__global__ void __launch_bounds__(256) reduce_partials_kernel(const double* __restrict__ partials, int nblk, int K, int K_out,
                                                              double* __restrict__ out, P2pPublish pub) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int k = warp; k < K_out; k += nw) {
    double s = 0.0;
    for (int b = lane; b < nblk; b += 32) s += partials[(size_t)b * K + k];
    s = warp_sum(s);
    if (lane == 0) {
      out[k] = s;
      if (pub.world) p2p_store(pub, k, s);
    }
  }
  if (pub.world) {
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) p2p_signal(pub);
  }
}

// publish K values that are already final on this rank (ranks without local paths, tests)
__global__ void p2p_publish_kernel(const double* __restrict__ vals, int K, P2pPublish pub) {
  for (int k = threadIdx.x; k < K; k += blockDim.x) p2p_store(pub, k, vals ? vals[k] : 0.0);
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) p2p_signal(pub);
}

// gather K values of the current epoch into out[] (tests; the product consumes them inside the payoff / finalize kernels)
__global__ void p2p_gather_kernel(P2pGather gat, int K, double* __restrict__ out) {
  for (int k = threadIdx.x; k < K; k += blockDim.x) out[k] = p2p_gather(gat, k);
}

// --------------------------------------------------------------------------------------------------------------------
// strict fixed-random steppers (parity entry points): reference evaluation order, no FMA contraction
// --------------------------------------------------------------------------------------------------------------------
struct LogsvRaw {
  double theta, kappa1, kappa2, beta, volvol, eta, alpha, adj, dt;
};

__global__ void __launch_bounds__(kThreads) logsv_step_fixed_kernel(double* __restrict__ x, double* __restrict__ sigma,
                                                                   double* __restrict__ qvar, const double* __restrict__ W0,
                                                                   const double* __restrict__ W1, int S, long long N, LogsvRaw r) {
  // pricers/logsv_pricer.py:1027-1047, expression by expression (fastmath=False in the reference)
  const double sdt = __dsqrt_rn(r.dt);
  const double vartheta2 = __dadd_rn(__dmul_rn(r.beta, r.beta), __dmul_rn(r.volvol, r.volvol));
  const double eta2 = __dmul_rn(r.eta, r.eta);
  const double k1theta = __dmul_rn(r.kappa1, r.theta);
  const double half_alpha = __dmul_rn(r.alpha, 0.5);
  const double half_vt2 = __dmul_rn(0.5, vartheta2);
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < N; i += stride) {
    double xi = x[i], si = sigma[i], qi = qvar[i];
    double L = log(si);
    for (int s = 0; s < S; ++s) {
      const double w0 = __dmul_rn(sdt, __ldg(W0 + (size_t)s * N + i));
      const double w1 = __dmul_rn(sdt, __ldg(W1 + (size_t)s * N + i));
      const double s2dt = __dmul_rn(__dmul_rn(__dmul_rn(eta2, si), si), r.dt);
      xi = __dadd_rn(__dadd_rn(xi, __dmul_rn(half_alpha, s2dt)), __dmul_rn(__dmul_rn(r.eta, si), w0));
      double d = __dadd_rn(__dadd_rn(__ddiv_rn(k1theta, si), -r.kappa1), __dmul_rn(r.kappa2, __dadd_rn(r.theta, -si)));
      d = __dadd_rn(__dadd_rn(d, __dmul_rn(r.adj, si)), -half_vt2);
      L = __dadd_rn(__dadd_rn(__dadd_rn(L, __dmul_rn(d, r.dt)), __dmul_rn(r.beta, w0)), __dmul_rn(r.volvol, w1));
      si = exp(L);
      qi = __dadd_rn(qi, __dmul_rn(0.5, __dadd_rn(s2dt, __dmul_rn(__dmul_rn(__dmul_rn(eta2, si), si), r.dt))));
    }
    x[i] = xi;
    sigma[i] = si;
    qvar[i] = qi;
  }
}

// Throughput variant of the fixed-random stepper for the device-resident calibration loop: same normals from HBM, but the
// per-step update of the fused kernel (LogsvPath<double>: folded constants, shared-polynomial exp pair, FMA) -- about half the
// fp64 instructions of the strict kernel, so the 16 B/path-step HBM stream becomes the bound.  Agrees with the strict kernel to
// ~1e-14 (tests/test_gpu_mc.py::test_device_resident_fixed_randoms_chain).
__global__ void __launch_bounds__(kThreads) logsv_step_fixed_fast_kernel(double* __restrict__ x, double* __restrict__ sigma,
                                                                        double* __restrict__ qvar, const double* __restrict__ W0,
                                                                        const double* __restrict__ W1, int S, long long N,
                                                                        LogsvConsts consts) {
  exp_table_init();
  LogsvPath<double> p(consts);
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < N; i += stride) {
    p.load(x[i], sigma[i], qvar[i]);
    for (int s = 0; s < S; ++s) p.step<true>(__ldg(W0 + (size_t)s * N + i), __ldg(W1 + (size_t)s * N + i));
    x[i] = p.x();
    sigma[i] = p.sigma();
    qvar[i] = p.q();
  }
}

__global__ void __launch_bounds__(kThreads) heston_step_fixed_kernel(double* __restrict__ x, double* __restrict__ var,
                                                                    double* __restrict__ qvar, const double* __restrict__ W0,
                                                                    const double* __restrict__ W1, int S, long long N,
                                                                    b200sv_heston_params p, double dt) {
  // pricers/heston_pricer.py:366-379
  const double sdt = __dsqrt_rn(dt);
  const double rho_1 = __dsqrt_rn(__dadd_rn(1.0, -__dmul_rn(p.rho, p.rho)));
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < N; i += stride) {
    double xi = x[i], vi = var[i], qi = qvar[i];
    for (int s = 0; s < S; ++s) {
      const double w0 = __dmul_rn(sdt, __ldg(W0 + (size_t)s * N + i));
      const double w1 = __dmul_rn(sdt, __ldg(W1 + (size_t)s * N + i));
      const double sig = __dsqrt_rn(vi);
      const double vdt = __dmul_rn(vi, dt);
      xi = __dadd_rn(__dadd_rn(xi, -__dmul_rn(0.5, vdt)), __dmul_rn(sig, w0));
      qi = __dadd_rn(qi, vdt);
      const double drift = __dmul_rn(__dmul_rn(p.kappa, __dadd_rn(p.theta, -vi)), dt);
      const double diff = __dmul_rn(__dmul_rn(sig, p.volvol), __dadd_rn(__dmul_rn(p.rho, w0), __dmul_rn(rho_1, w1)));
      vi = __dadd_rn(__dadd_rn(vi, drift), diff);
      vi = vi < 1e-4 ? 1e-4 : vi;   // np.maximum(var0, 1e-4): NaN stays NaN
    }
    x[i] = xi;
    var[i] = vi;
    qvar[i] = qi;
  }
}

// Full volatility paths sigma_t[(S+1)][N]: simulate_vol_paths (pricers/logsv_pricer.py:870-947).  One normal per step
// (vartheta * w1), drift evaluated at the current step, reference evaluation order (it is plain numpy, no fastmath).
// W != nullptr: caller-supplied SCALED increments [S][N] ("brownians"); else sqrt(dt) * Z0 of the device Philox stream
// (gauss f64: call = step, first normal of the pair).  Output-bandwidth bound: 8 B written per path-step.
__global__ void __launch_bounds__(kThreads) logsv_vol_paths_kernel(double* __restrict__ sigma_t, const double* __restrict__ W, int S,
                                                                  long long N, LogsvRaw r, double v0, unsigned long long seed,
                                                                  unsigned long long path_offset) {
  const double sdt = __dsqrt_rn(r.dt);
  const double vartheta2 = __dadd_rn(__dmul_rn(r.beta, r.beta), __dmul_rn(r.volvol, r.volvol));
  const double vartheta = __dsqrt_rn(vartheta2);
  const double k1theta = __dmul_rn(r.kappa1, r.theta);
  const double half_vt2 = __dmul_rn(0.5, vartheta2);
  gauss64_table_init();
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < N; i += stride) {
    double si = v0;
    double L = log(si);
    sigma_t[i] = si;
    StepNormals<double, kGaussF64> rng(seed, path_offset + (unsigned long long)i, 0u);
    for (int s = 0; s < S; ++s) {
      double w1;
      if (W) {
        w1 = __ldg(W + (size_t)s * N + i);
      } else {
        double z0, z1;
        rng.get((uint32_t)s, z0, z1);
        w1 = __dmul_rn(sdt, z0);
      }
      double d = __dadd_rn(__dadd_rn(__ddiv_rn(k1theta, si), -r.kappa1), __dmul_rn(r.kappa2, __dadd_rn(r.theta, -si)));
      d = __dadd_rn(__dadd_rn(d, __dmul_rn(r.adj, si)), -half_vt2);
      L = __dadd_rn(__dadd_rn(L, __dmul_rn(d, r.dt)), __dmul_rn(vartheta, w1));
      si = exp(L);
      sigma_t[(size_t)(s + 1) * N + i] = si;
    }
  }
}

// (sum F e^x over non-NaN, count) partials for externally supplied states (b200sv_mc_payoffs)
__global__ void __launch_bounds__(kThreads) spot_moments_kernel(const double* __restrict__ x, long long n, double forward,
                                                               double* __restrict__ partials) {
  SpotMoments<2, kThreads> mom;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) mom.add(forward * exp(x[i]));
  mom.store(partials);
}

// --------------------------------------------------------------------------------------------------------------------
// payoff sums: utils/mc_payoffs.py:61-88
// --------------------------------------------------------------------------------------------------------------------
// The strikes and payoff codes of the C strikes from j0 on; a slot past the slice's J strikes has ty = -1
template <int C>
__device__ __forceinline__ void load_strike_chunk(const double* __restrict__ strikes, const int8_t* __restrict__ types, int J, int j0,
                                                  double (&kk)[C], int (&ty)[C]) {
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const int j = j0 + c;
    kk[c] = j < J ? strikes[j] : 0.0;
    ty[c] = j < J ? (int)types[j] : -1;
  }
}

// General payoffs (any mix of C / P / IC / IP): per-strike NaN-skipping counts, IEEE division for the inverse payoffs.
// payoff_general_block / payoff_vanilla_block: the work of ONE CTA for the strike chunk starting at j0 -- grid-stride over the paths with
// `nblocks` CTAs, block-reduce, write this CTA's partial row.  Called by the stand-alone payoff kernels (blockIdx.y = chunk) and by the
// cooperative whole-chain kernel (chunks looped inside).
template <typename Real>
__device__ __forceinline__ void payoff_general_block(const Real* __restrict__ x, const Real* __restrict__ q, long long n, double ttm, double forward,
                                                     const double* __restrict__ strikes, const int8_t* __restrict__ types, int J, int variable_type,
                                                     double corr, double* __restrict__ partials, int Kpad, int j0, int block, int nblocks) {
  __shared__ double red[3 * kStrikeChunk * kThreads / 32];
  double kk[kStrikeChunk];
  int ty[kStrikeChunk];
  load_strike_chunk(strikes, types, J, j0, kk, ty);
  const bool is_qvar = variable_type == B200SV_Q_VAR;
  double acc[3 * kStrikeChunk];
#pragma unroll
  for (int c = 0; c < 3 * kStrikeChunk; ++c) acc[c] = 0.0;
  const long long stride = (long long)nblocks * kThreads;
  for (long long i = (long long)block * kThreads + threadIdx.x; i < n; i += stride) {
    const double spot = forward * exp((double)x[i]) - corr;
    const double under = is_qvar ? (double)q[i] / ttm : spot;
#pragma unroll
    for (int c = 0; c < kStrikeChunk; ++c) {
      if (ty[c] >= 0) {
        const bool is_put = (ty[c] & 1);
        double pay = is_put ? (under < kk[c] ? kk[c] - under : 0.0) : (under > kk[c] ? under - kk[c] : 0.0);
        // np.where(np.greater(nan, k), ..., 0.0) == 0.0: a NaN underlying pays 0 for C/P and 0/NaN = NaN (skipped) for IC/IP
        if (ty[c] >= 2) pay = pay / spot;
        if (pay == pay) {
          acc[3 * c + 0] += pay;
          acc[3 * c + 1] += pay * pay;
          acc[3 * c + 2] += 1.0;
        }
      }
    }
  }
  block_sum<3 * kStrikeChunk, kThreads>(acc, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int c = 0; c < 3 * kStrikeChunk; ++c) partials[(size_t)block * Kpad + 3 * j0 + c] = acc[c];
  }
}

// Vanilla-only payoffs ('C' / 'P' in every slot of the slice): pay = max(+-(U - K), 0) is never NaN (numpy's
// where(greater(nan, K), ., 0.0) is 0.0 as well), so every path counts and the count is simply n; no division, no branches.
// ~6 instructions per (path, strike) + one exp per (path, chunk); kPayoffUnroll loads in flight per thread.
constexpr int kPayoffUnroll = 4;
template <typename Real>
__device__ __forceinline__ void payoff_vanilla_block(const Real* __restrict__ x, const Real* __restrict__ q, long long n, double ttm, double forward,
                                                     const double* __restrict__ strikes, const int8_t* __restrict__ types, int J, int variable_type,
                                                     double corr, double* __restrict__ partials, int Kpad, int j0, int block, int nblocks) {
  __shared__ double red[2 * kStrikeChunk * kThreads / 32];
  double sg[kStrikeChunk], nk[kStrikeChunk];      // pay = max(sg*U + nk, 0), nk = -sg*K
#pragma unroll
  for (int c = 0; c < kStrikeChunk; ++c) {
    const int j = j0 + c;
    const double sgn = (j < J && (types[j] & 1)) ? -1.0 : 1.0;
    sg[c] = sgn;
    nk[c] = j < J ? -sgn * strikes[j] : -INFINITY;   // unused slot: max(U - inf, 0) = 0
  }
  const bool is_qvar = variable_type == B200SV_Q_VAR;
  const double inv_ttm = 1.0 / ttm;
  double acc[2 * kStrikeChunk];
#pragma unroll
  for (int c = 0; c < 2 * kStrikeChunk; ++c) acc[c] = 0.0;
  auto accumulate = [&](double under) {
#pragma unroll
    for (int c = 0; c < kStrikeChunk; ++c) {
      const double d = fma(sg[c], under, nk[c]);
      const double pay = d > 0.0 ? d : 0.0;
      acc[2 * c] += pay;
      acc[2 * c + 1] = fma(pay, pay, acc[2 * c + 1]);
    }
  };
  const long long stride = (long long)nblocks * kThreads;
  long long i = (long long)block * kThreads + threadIdx.x;
  if (!is_qvar) {
    for (; i + (kPayoffUnroll - 1) * stride < n; i += kPayoffUnroll * stride) {
      double xs[kPayoffUnroll];
#pragma unroll
      for (int u = 0; u < kPayoffUnroll; ++u) xs[u] = (double)x[i + u * stride];
#pragma unroll
      for (int u = 0; u < kPayoffUnroll; ++u) accumulate(forward * exp(xs[u]) - corr);
    }
    for (; i < n; i += stride) accumulate(forward * exp((double)x[i]) - corr);
  } else {
    for (; i < n; i += stride) accumulate((double)q[i] * inv_ttm);
  }
  block_sum<2 * kStrikeChunk, kThreads>(acc, red);
  if (threadIdx.x == 0) {
    // count of paths this CTA visited (same for every strike)
    const long long first = (long long)block * kThreads;
    long long cnt = 0;
    if (first < n) {
      const long long full_rounds = (n - first) / stride, rem = (n - first) % stride;
      cnt = full_rounds * kThreads + (rem < kThreads ? rem : kThreads);
    }
#pragma unroll
    for (int c = 0; c < kStrikeChunk; ++c) {
      partials[(size_t)block * Kpad + 3 * (j0 + c) + 0] = acc[2 * c];
      partials[(size_t)block * Kpad + 3 * (j0 + c) + 1] = acc[2 * c + 1];
      partials[(size_t)block * Kpad + 3 * (j0 + c) + 2] = (double)cnt;
    }
  }
}

// correnction = np.nanmean(spots_t) - forward; multi-GPU: the GLOBAL (sum, count) is gathered from the peers' mailbox writes here
__device__ __forceinline__ double payoff_recentring(const double* __restrict__ moments, double forward, const P2pGather& gat) {
  __shared__ double sh_mom[2];
  if (threadIdx.x < 2) sh_mom[threadIdx.x] = gat.world ? p2p_gather(gat, threadIdx.x) : moments[threadIdx.x];
  __syncthreads();
  return sh_mom[0] / sh_mom[1] - forward;
}

template <typename Real>
__global__ void __launch_bounds__(kThreads) payoff_kernel(const Real* __restrict__ x, const Real* __restrict__ q, long long n,
                                                         double ttm, double forward, const double* __restrict__ strikes,
                                                         const int8_t* __restrict__ types, int J, int variable_type,
                                                         const double* __restrict__ moments, double* __restrict__ partials,
                                                         int Kpad /* = 3 * kStrikeChunk * gridDim.y */, P2pGather gat) {
  const double corr = payoff_recentring(moments, forward, gat);
  payoff_general_block<Real>(x, q, n, ttm, forward, strikes, types, J, variable_type, corr, partials, Kpad, blockIdx.y * kStrikeChunk, blockIdx.x, gridDim.x);
}

template <typename Real>
__global__ void __launch_bounds__(kThreads) payoff_vanilla_kernel(const Real* __restrict__ x, const Real* __restrict__ q, long long n,
                                                                 double ttm, double forward, const double* __restrict__ strikes,
                                                                 const int8_t* __restrict__ types, int J, int variable_type,
                                                                 const double* __restrict__ moments, double* __restrict__ partials,
                                                                 int Kpad, P2pGather gat) {
  const double corr = payoff_recentring(moments, forward, gat);
  payoff_vanilla_block<Real>(x, q, n, ttm, forward, strikes, types, J, variable_type, corr, partials, Kpad, blockIdx.y * kStrikeChunk, blockIdx.x, gridDim.x);
}

// optional fused Black-76 inversion of the prices just assembled (batched calibration objective): needs strikes/types/forward/ttm
struct IvolSpec {
  const double* strikes;
  const int8_t* types;
  double forward, ttm;
  double* ivols;       // nullptr: skip
};

__global__ void payoff_finalize_kernel(const double* __restrict__ sums, int J, double discfactor, double total_paths,
                                       double* __restrict__ prices, double* __restrict__ stderrs, P2pGather gat, IvolSpec iv = IvolSpec{}) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= J) return;
  const double s1 = gat.world ? p2p_gather(gat, 3 * j) : sums[3 * j];
  const double s2 = gat.world ? p2p_gather(gat, 3 * j + 1) : sums[3 * j + 1];
  const double cnt = gat.world ? p2p_gather(gat, 3 * j + 2) : sums[3 * j + 2];
  const double mean = s1 / cnt;
  double var = s2 / cnt - mean * mean;
  var = var < 0.0 ? 0.0 : var;                                 // a NaN variance (infinite payoff sums) stays NaN, as in np.nanstd
  prices[j] = discfactor * mean;                               // discfactor*np.nanmean(payoff)
  stderrs[j] = discfactor * sqrt(var) / sqrt(total_paths);     // discfactor*np.nanstd(payoff) / sqrt(x0.shape[0])
  if (iv.ivols) iv.ivols[j] = black_implied_vol(iv.forward, iv.strikes[j], iv.ttm, discfactor, discfactor * mean, iv.types[j]);
}

// --------------------------------------------------------------------------------------------------------------------
// the whole chain in ONE persistent cooperative kernel (single GPU, fp64 state)
// --------------------------------------------------------------------------------------------------------------------
// north_star: "one persistent-thread kernel ... with a warp-shuffle block reduction of terminal payoffs into per-strike sums/sum-squares
// staged in shared memory".  The forward re-centring of utils/mc_payoffs.py:61-63 needs the mean over ALL paths before any payoff, so
// a chain is two grid-wide phases per maturity; here they are separated by grid.sync() instead of kernel boundaries:
//   for every maturity:  slice phase (Philox + stepper, state in registers, per-CTA moments)  -> grid.sync
//                        every CTA reduces the per-CTA moments in the same fixed order -> correction; payoff phase (per-CTA per-strike
//                        partial sums, the same block functions as the stand-alone payoff kernels)               -> grid.sync
//                        CTA j (j < J) reduces column j over the CTAs in fixed order and finalises price / std error / implied vol
// One launch instead of 5 per maturity: a 4-maturity chain at 1e4 paths drops from 0.24 ms to the latency of the dependent steps.
// The grid is one co-resident wave (cudaLaunchCooperativeKernel); buffers are reused across maturities -- the two syncs order every
// write after the last read of the previous use (a CTA cannot pass sync k+1 before every CTA has arrived, i.e. finished reading).
template <typename Consts>
struct CoopSliceSpec {
  Consts c;
  int nsteps, jo, J, kinds;
  double forward, ttm, discfactor;
};

struct CoopArgs {
  double *x, *v, *q;              // state SoA [n]
  long long n;
  double v_init;
  unsigned long long seed;
  int M, variable_type;
  const double* strikes;          // [Jtot]
  const int8_t* types;
  double* part_mom;               // [grid][2]
  double* part_pay;               // [grid][Kpad_max]
  int Kpad_max;
  double total_paths;
  double *prices, *stderrs, *ivols;   // [Jalloc] each; ivols may be nullptr
};

template <typename Path, typename Consts, int GAUSS>
__global__ void __launch_bounds__(kSliceThreads, B200SV_SLICE_MINBLOCKS) mc_chain_coop_kernel(CoopArgs a, const CoopSliceSpec<Consts>* __restrict__ specs) {
  static_assert(kSliceThreads == kThreads, "the payoff block functions and the slice phase share one CTA size");
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  __shared__ double red[2 * kSliceThreads / 32];
  __shared__ double sh_corr;
  exp_table_init();
  if constexpr (GAUSS != kGaussF32) gauss64_table_init();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long stride = (long long)gridDim.x * kSliceThreads;
  for (int m = 0; m < a.M; ++m) {
    const CoopSliceSpec<Consts> sp = specs[m];
    // ---- slice phase ------------------------------------------------------------------------------------------------------------
    {
      double acc[2] = {0.0, 0.0};
      Path p(sp.c);
      const SliceArgs<double> s{a.x, a.v, a.q, a.n, 0ull, m == 0, a.v_init, sp.nsteps, (unsigned int)m, a.seed, sp.forward, a.part_mom};
      for (long long i = (long long)blockIdx.x * kSliceThreads + threadIdx.x; i < a.n; i += stride) {
        const double xT = slice_path<Path, double, GAUSS>(p, s, i);
        const double spot = sp.forward * exp(xT);
        if (spot == spot) {
          acc[0] += spot;
          acc[1] += 1.0;
        }
      }
      block_sum<2, kSliceThreads>(acc, red);
      if (threadIdx.x == 0) {
        a.part_mom[2 * blockIdx.x + 0] = acc[0];
        a.part_mom[2 * blockIdx.x + 1] = acc[1];
      }
    }
    if (sp.J == 0) {           // nothing to price at this maturity: the state is stored, go on (uniform across the grid: no sync imbalance)
      grid.sync();
      continue;
    }
    grid.sync();
    // ---- global moments (same fixed order in every CTA: lanes stride over the CTAs, shuffle tree) -> correction ----------------------
    if (warp == 0) {
      double s0 = 0.0, s1 = 0.0;
      for (int b = lane; b < (int)gridDim.x; b += 32) {
        s0 += __ldcg(a.part_mom + 2 * b);
        s1 += __ldcg(a.part_mom + 2 * b + 1);
      }
      s0 = warp_sum(s0);
      s1 = warp_sum(s1);
      if (lane == 0) sh_corr = s0 / s1 - sp.forward;
    }
    __syncthreads();
    const double corr = sh_corr;
    // ---- payoff phase ---------------------------------------------------------------------------------------------------------------
    const int chunks = (sp.J + kStrikeChunk - 1) / kStrikeChunk;
    const int Kpad = 3 * kStrikeChunk * chunks;
    for (int ch = 0; ch < chunks; ++ch) {
      if (sp.kinds == 1)
        payoff_vanilla_block<double>(a.x, a.q, a.n, sp.ttm, sp.forward, a.strikes + sp.jo, a.types + sp.jo, sp.J, a.variable_type, corr, a.part_pay, Kpad,
                                     ch * kStrikeChunk, blockIdx.x, gridDim.x);
      else
        payoff_general_block<double>(a.x, a.q, a.n, sp.ttm, sp.forward, a.strikes + sp.jo, a.types + sp.jo, sp.J, a.variable_type, corr, a.part_pay, Kpad,
                                     ch * kStrikeChunk, blockIdx.x, gridDim.x);
    }
    grid.sync();
    // ---- finalise: strike j by CTA j % grid (warp 0), fixed-order sum over the CTAs ---------------------------------------------------
    for (int j = blockIdx.x; j < sp.J; j += gridDim.x) {
      if (warp == 0) {
        double s1 = 0.0, s2 = 0.0, cnt = 0.0;
        for (int b = lane; b < (int)gridDim.x; b += 32) {
          const double* row = a.part_pay + (size_t)b * Kpad + 3 * j;
          s1 += __ldcg(row);
          s2 += __ldcg(row + 1);
          cnt += __ldcg(row + 2);
        }
        s1 = warp_sum(s1);
        s2 = warp_sum(s2);
        cnt = warp_sum(cnt);
        if (lane == 0) {
          const double mean = s1 / cnt;
          double var = s2 / cnt - mean * mean;
          var = var > 0.0 ? var : 0.0;
          a.prices[sp.jo + j] = sp.discfactor * mean;
          a.stderrs[sp.jo + j] = sp.discfactor * sqrt(var) / sqrt(a.total_paths);
          if (a.ivols)
            a.ivols[sp.jo + j] = black_implied_vol(sp.forward, a.strikes[sp.jo + j], sp.ttm, sp.discfactor, sp.discfactor * mean, a.types[sp.jo + j]);
        }
      }
    }
    // the next maturity's slice phase overwrites part_mom only: every CTA has read it before arriving at the sync above
  }
}

// --------------------------------------------------------------------------------------------------------------------
// pathwise (forward-mode) sensitivities of the chain pricer, DESIGN.md §3.9
// --------------------------------------------------------------------------------------------------------------------
// A tangent path wraps the production path object and calls its step() unchanged, so the base recursion -- and the prices -- are the
// same code as mc_slice_kernel's.  Per model parameter p it carries, in registers, the tangent of the vol state (dL = d log sigma for
// LogSV, dv for Heston) and two running sums from which the tangents of x and q follow.  Parameter order = the dataclass field order.
constexpr int kLogsvParams = 6;    // sigma0, theta, kappa1, kappa2, beta, volvol
constexpr int kHestonParams = 5;   // v0, theta, kappa, rho, volvol

struct TangentState {    // SoA [P][n] fp64, persisted across maturities like x, v, q
  double* dx;
  double* dv;            // d log sigma (LogSV) or d variance (Heston)
  double* dq;
};

struct LogsvTangentConsts {
  LogsvConsts c;
  double a1, a2;                     // natural-unit a1, a2 of LogsvConsts (the recursion's Jacobian 1 - a1/sigma + a2*sigma)
  double cx2, cq4;                   // 2 cx, 4 cq
  double dt, sdt, k1dt, k2dt, thdt, bdt, vvdt, etadt;   // parameter derivatives of a0..b1 (etadt = eta*dt under the inverse measure, else 0)
};

struct HestonTangentConsts {
  HestonConsts c;
  double drc0, drc1, dvc0, dvc1;     // d(c0, c1)/d rho, d(c0, c1)/d volvol
};

static LogsvTangentConsts make_logsv_tangent_consts(const b200sv_logsv_params& p, double eta, bool spot, double dt) {
  LogsvTangentConsts k;
  k.c = make_logsv_consts(p, eta, spot, dt);
  k.a1 = k.c.a1;
  k.a2 = k.c.a2;
  k.cx2 = 2.0 * k.c.cx;
  k.cq4 = 4.0 * k.c.cq;
  k.dt = dt;
  k.sdt = std::sqrt(dt);
  k.k1dt = p.kappa1 * dt;
  k.k2dt = p.kappa2 * dt;
  k.thdt = p.theta * dt;
  k.bdt = p.beta * dt;
  k.vvdt = p.volvol * dt;
  k.etadt = spot ? 0.0 : eta * dt;
  return k;
}

static HestonTangentConsts make_heston_tangent_consts(const b200sv_heston_params& p, double dt) {
  HestonTangentConsts k;
  k.c = make_heston_consts(p, dt, B200SV_HESTON_EULER_FLOOR);
  const double sdt = std::sqrt(dt), r1 = std::sqrt(1.0 - p.rho * p.rho);
  k.drc0 = p.volvol * sdt;
  k.drc1 = -p.volvol * p.rho / r1 * sdt;
  k.dvc0 = p.rho * sdt;
  k.dvc1 = r1 * sdt;
  return k;
}

// LogSV: dL' = dL (1 - a1/sigma + a2 sigma) + da0 + da1/sigma + da2 sigma + db0 z0 + db1 z1 on the OLD sigma;
// dx += (2 cx sigma^2 + ce sigma z0) dL on the old sigma; dq is kept as dq0 + 2 cq sigma_0^2 dL_0 + sum_k 4 cq sigma_k^2 dL_k (new sigma
// of every step) and corrected by -2 cq sigma_S^2 dL_S when read, the same telescoping as LogsvPath's q.
struct LogsvTangentPath {
  static constexpr int NP = kLogsvParams;
  static constexpr bool kPrefetch = false;   // 18 tangent registers leave no room for a second set of normals in flight
  static constexpr bool kRecordsLastStep = false;
  using Consts = LogsvTangentConsts;
  LogsvPath<double> b;
  double dx[NP], dL[NP], dq[NP];
  double s_first;      // sigma at load
  const Consts& k;     // the kernel's __grid_constant__ parameter: read as constant-bank operands, not held in registers
  __device__ __forceinline__ LogsvTangentPath(const Consts& k_) : b(k_.c), k(k_) {}
  __device__ __forceinline__ void load(double x, double v, double q, const TangentState& t, long long i, long long n, bool init) {
    b.load(x, v, q);
    s_first = v;
#pragma unroll
    for (int p = 0; p < NP; ++p) {
      double tx = 0.0, tl = (p == 0) ? 1.0 / v : 0.0, tq = 0.0;    // dL_0 = 1/sigma0 for sigma0
      if (!init) {
        tx = t.dx[p * n + i];
        tl = t.dv[p * n + i];
        tq = t.dq[p * n + i];
      }
      dx[p] = tx;
      dL[p] = tl;
      dq[p] = fma(2.0 * k.c.cq * b.s2_first, tl, tq);
    }
  }
  template <bool SAFE>
  __device__ __forceinline__ void step(double z0, double z1) {
    const double so = b.s, io = b.inv;
    b.template step<SAFE>(z0, z1);
    const double sn = b.s;
    const double jac = fma(k.a2, so, fma(-k.a1, io, 1.0));
    const double fx = so * fma(k.cx2, so, k.c.ce * z0);
    const double fq = k.cq4 * sn * sn;
    double drive[NP];
    drive[0] = 0.0;
    drive[1] = fma(k.k1dt, io, k.k2dt);                      // theta:  kappa2 dt + kappa1 dt / sigma
    drive[2] = fma(k.thdt, io, -k.dt);                       // kappa1: -dt + theta dt / sigma
    drive[3] = fma(-k.dt, so, k.thdt);                       // kappa2: theta dt - dt sigma
    drive[4] = fma(k.sdt, z0, fma(k.etadt, so, -k.bdt));     // beta:   -beta dt + eta dt sigma (inverse measure) + sqrt(dt) z0
    drive[5] = fma(k.sdt, z1, -k.vvdt);                      // volvol: -volvol dt + sqrt(dt) z1
    // a clamped step (SAFE re-run of a path that left the representable range) has a zero tangent through the clamp
    const bool clamped = SAFE && fabs(b.Ls) == kLogScaledMax;
#pragma unroll
    for (int p = 0; p < NP; ++p) {
      dx[p] = fma(fx, dL[p], dx[p]);
      dL[p] = clamped ? 0.0 : fma(jac, dL[p], drive[p]);
      dq[p] = fma(fq, dL[p], dq[p]);
    }
  }
  __device__ __forceinline__ bool overflowed() const { return b.overflowed(); }
  __device__ __forceinline__ double sigma() const { return b.sigma(); }
  // LogsvPath::x() / q() with the contraction nvcc applies to them in every production kernel spelled out -- s2_first - s*s is
  // fma(sigma_0, sigma_0, -rn(s*s)) there -- so that the state stays bit-identical to mc_slice_kernel's in this different context
  __device__ __forceinline__ double s2_diff() const { return fma(s_first, s_first, -__dmul_rn(b.s, b.s)); }
  __device__ __forceinline__ double x() const { return fma(b.ce, b.XM, fma(b.cx, s2_diff() + b.A, b.x0)); }
  __device__ __forceinline__ double q() const { return fma(b.cq, s2_diff() + 2.0 * b.A, b.q0); }
  __device__ __forceinline__ double tx(int p) const { return dx[p]; }
  __device__ __forceinline__ double tq(int p) const { return fma(-2.0 * k.c.cq * b.s * b.s, dL[p], dq[p]); }
  __device__ __forceinline__ double tv(int p) const { return dL[p]; }
  // the vol state a step reads (old sigma) and the standard deviation ce sigma of that step's log-spot increment
  __device__ __forceinline__ double step_vol() const { return b.s; }
  __device__ __forceinline__ double step_sd(double vol) const { return b.ce * vol; }
};

// Heston floor-Euler: dv' = 0 where the floor binds, else dv (1 - kappa dt) + dv (c0 z0 + c1 z1)/(2 sqrt v) + d(kappa dt) (theta - v)
// + kappa dt d(theta) + sqrt(v) (dc0 z0 + dc1 z1); dx += (-dt/2 + sqrt(dt) z0 / (2 sqrt v)) dv, dq += dt dv, all on the old v.
struct HestonTangentPath {
  static constexpr int NP = kHestonParams;
  static constexpr bool kPrefetch = B200SV_SLICE_PREFETCH != 0;
  static constexpr bool kRecordsLastStep = false;
  using Consts = HestonTangentConsts;
  HestonPath<double, false> b;
  double dx[NP], dv[NP], dq[NP];
  const Consts& k;     // the kernel's __grid_constant__ parameter
  __device__ __forceinline__ HestonTangentPath(const Consts& k_) : b(k_.c), k(k_) {}
  __device__ __forceinline__ void load(double x, double v, double q, const TangentState& t, long long i, long long n, bool init) {
    b.load(x, v, q);
#pragma unroll
    for (int p = 0; p < NP; ++p) {
      if (init) {
        dx[p] = 0.0;
        dv[p] = (p == 0) ? 1.0 : 0.0;                    // dv_0 = 1 for v0
        dq[p] = 0.0;
      } else {
        dx[p] = t.dx[p * n + i];
        dv[p] = t.dv[p * n + i];
        dq[p] = t.dq[p * n + i];
      }
    }
  }
  template <bool SAFE>
  __device__ __forceinline__ void step(double z0, double z1) {
    const double v = b.v, sig = sqrt(v), hs = 0.5 / sig;
    b.template step<SAFE>(z0, z1);
    const bool live = b.v > 1e-4;                        // np.maximum(v, 1e-4) did not bind
    const double fx = fma(b.sdt * z0, hs, b.hx);
    const double jac = fma(fma(b.c0, z0, b.c1 * z1), hs, 1.0 - b.kdt);
    double drive[NP];
    drive[0] = 0.0;
    drive[1] = b.kdt;                                    // theta
    drive[2] = b.dt * (b.theta - v);                     // kappa
    drive[3] = sig * fma(k.drc0, z0, k.drc1 * z1);       // rho
    drive[4] = sig * fma(k.dvc0, z0, k.dvc1 * z1);       // volvol
#pragma unroll
    for (int p = 0; p < NP; ++p) {
      dx[p] = fma(fx, dv[p], dx[p]);
      dq[p] = fma(b.dt, dv[p], dq[p]);
      dv[p] = live ? fma(jac, dv[p], drive[p]) : 0.0;
    }
  }
  __device__ __forceinline__ bool overflowed() const { return false; }
  __device__ __forceinline__ double sigma() const { return b.sigma(); }
  __device__ __forceinline__ double x() const { return b.x(); }
  __device__ __forceinline__ double q() const { return b.q(); }
  __device__ __forceinline__ double tx(int p) const { return dx[p]; }
  __device__ __forceinline__ double tq(int p) const { return dq[p]; }
  __device__ __forceinline__ double tv(int p) const { return dv[p]; }
  // the vol state a step reads (old variance) and the standard deviation sqrt(v dt) of that step's log-spot increment
  __device__ __forceinline__ double step_vol() const { return b.v; }
  __device__ __forceinline__ double step_sd(double vol) const { return b.sdt * sqrt(vol); }
};

// Monte Carlo gamma (DESIGN.md §3.9): TPath that also keeps the vol state and z0 of the step in flight, so that after the slice the
// conditional law of the last log-spot step is known -- x_S = mu + s z0_S with s = step_sd(vol_{S-1}) -- and writes (s, mu) to
// laststep [2][n].  z0 is the value the step consumed (after the float-to-double conversion of the fp32 stream); the overflow re-run
// replays every step, so the recorded step is the clamped one where the path was re-run.
template <typename TPath>
struct LastStepConsts {
  typename TPath::Consts c;
  double* laststep;
};

template <typename TPath>
struct LastStepPath : TPath {
  using Consts = LastStepConsts<TPath>;
  static constexpr bool kRecordsLastStep = true;
  double vol_last, z_last;
  double* out;
  __device__ __forceinline__ LastStepPath(const Consts& k_) : TPath(k_.c), out(k_.laststep) {}
  template <bool SAFE>
  __device__ __forceinline__ void step(double z0, double z1) {
    vol_last = TPath::step_vol();
    z_last = z0;
    TPath::template step<SAFE>(z0, z1);
  }
  __device__ __forceinline__ void record_last_step(long long i, long long n, double xT) const {
    const double s = TPath::step_sd(vol_last);
    out[i] = s;
    out[n + i] = fma(-s, z_last, xT);
  }
};

// Monte Carlo theta (DESIGN.md §3.12): the one tangent direction d/d dt of a slice's step length, its step count S held, starting at 0 at
// the slice's first step (the state at ttms[m - 1] does not depend on ttms[m]).  Every step constant is proportional to dt or sqrt(dt), so
// its explicit derivative is c / dt or c / (2 dt); the *d members below hold those.  tq() hands the payoff kernel dq - qshift q with
// qshift = S / ttm: the Q_VAR underlying is q / ttm and ttm moves by S per unit dt, so its derivative is tq() / ttm with no payoff branch.
struct LogsvThetaConsts {
  LogsvConsts c;
  double a1, a2;                     // natural-unit a1, a2 (the recursion's Jacobian 1 - a1/sigma + a2*sigma)
  double cx2, cq2;                   // 2 cx, 2 cq
  double a0d, a1d, a2d, b0h, b1h;    // a0/dt, a1/dt, a2/dt, b0/(2dt), b1/(2dt)
  double cxd, ceh, cqd;              // cx/dt, ce/(2dt), cq/dt
  double qshift;
};

struct HestonThetaConsts {
  HestonConsts c;
  double kappa, hdt, hsdt;           // kappa, 1/(2dt), 1/(2 sqrt(dt))
  double qshift;
};

static LogsvThetaConsts make_logsv_theta_consts(const b200sv_logsv_params& p, double eta, bool spot, double dt, double qshift) {
  LogsvThetaConsts k;
  k.c = make_logsv_consts(p, eta, spot, dt);
  k.a1 = k.c.a1;
  k.a2 = k.c.a2;
  k.cx2 = 2.0 * k.c.cx;
  k.cq2 = 2.0 * k.c.cq;
  k.a0d = k.c.a0 / dt;
  k.a1d = k.c.a1 / dt;
  k.a2d = k.c.a2 / dt;
  k.b0h = 0.5 * k.c.b0 / dt;
  k.b1h = 0.5 * k.c.b1 / dt;
  k.cxd = k.c.cx / dt;
  k.ceh = 0.5 * k.c.ce / dt;
  k.cqd = k.c.cq / dt;
  k.qshift = qshift;
  return k;
}

static HestonThetaConsts make_heston_theta_consts(const b200sv_heston_params& p, double dt, double qshift) {
  HestonThetaConsts k;
  k.c = make_heston_consts(p, dt, B200SV_HESTON_EULER_FLOOR);
  k.kappa = p.kappa;
  k.hdt = 0.5 / dt;
  k.hsdt = 0.5 / std::sqrt(dt);
  k.qshift = qshift;
  return k;
}

// LogSV, on the old sigma:  dL' = dL (1 - a1/sigma + a2 sigma) + (a0 + a1/sigma + a2 sigma)/dt + (b0 z0 + b1 z1)/(2dt), 0 through a clamp;
// dx += (2 cx sigma^2 + ce sigma z0) dL + (cx sigma^2 + ce sigma z0 / 2)/dt;  dq += 2 cq (sigma^2 dL + sigma'^2 dL') + cq (sigma^2 + sigma'^2)/dt
struct LogsvThetaPath {
  static constexpr int NP = 1;
  static constexpr bool kPrefetch = B200SV_SLICE_PREFETCH != 0;
  static constexpr bool kRecordsLastStep = false;
  using Consts = LogsvThetaConsts;
  LogsvPath<double> b;
  double dx, dL, dq;
  double s_first;
  const Consts& k;     // the kernel's __grid_constant__ parameter
  __device__ __forceinline__ LogsvThetaPath(const Consts& k_) : b(k_.c), k(k_) {}
  __device__ __forceinline__ void load(double x, double v, double q, const TangentState&, long long, long long, bool) {
    b.load(x, v, q);
    s_first = v;
    dx = dL = dq = 0.0;
  }
  template <bool SAFE>
  __device__ __forceinline__ void step(double z0, double z1) {
    const double so = b.s, io = b.inv;
    b.template step<SAFE>(z0, z1);
    const double sn = b.s, so2 = so * so, sn2 = sn * sn;
    const double jac = fma(k.a2, so, fma(-k.a1, io, 1.0));
    const double drive = fma(k.b0h, z0, fma(k.b1h, z1, fma(k.a2d, so, fma(k.a1d, io, k.a0d))));
    const double sz = so * z0;
    dx = fma(so * fma(k.cx2, so, k.c.ce * z0), dL, dx) + fma(k.cxd, so2, k.ceh * sz);
    const bool clamped = SAFE && fabs(b.Ls) == kLogScaledMax;
    const double dLn = clamped ? 0.0 : fma(jac, dL, drive);
    dq += fma(k.cq2, fma(so2, dL, sn2 * dLn), k.cqd * (so2 + sn2));
    dL = dLn;
  }
  __device__ __forceinline__ bool overflowed() const { return b.overflowed(); }
  __device__ __forceinline__ double sigma() const { return b.sigma(); }
  // LogsvTangentPath::x() / q(): the production kernels' contraction spelled out
  __device__ __forceinline__ double s2_diff() const { return fma(s_first, s_first, -__dmul_rn(b.s, b.s)); }
  __device__ __forceinline__ double x() const { return fma(b.ce, b.XM, fma(b.cx, s2_diff() + b.A, b.x0)); }
  __device__ __forceinline__ double q() const { return fma(b.cq, s2_diff() + 2.0 * b.A, b.q0); }
  __device__ __forceinline__ double tx(int) const { return dx; }
  __device__ __forceinline__ double tq(int) const { return fma(-k.qshift, q(), dq); }
  __device__ __forceinline__ double tv(int) const { return dL; }
};

// Heston floor-Euler, on the old v:  dv' = dv (1 - kappa dt) + kappa (theta - v) + dv (c0 z0 + c1 z1)/(2 sqrt v) + sqrt(v) (c0 z0 + c1 z1)/(2dt),
// 0 where the floor binds;  dx += (-dt/2 + sqrt(dt) z0 / (2 sqrt v)) dv - v/2 + sqrt(v) z0 / (2 sqrt dt);  dq += dt dv + v
struct HestonThetaPath {
  static constexpr int NP = 1;
  static constexpr bool kPrefetch = B200SV_SLICE_PREFETCH != 0;
  static constexpr bool kRecordsLastStep = false;
  using Consts = HestonThetaConsts;
  HestonPath<double, false> b;
  double dx, dv, dq;
  const Consts& k;     // the kernel's __grid_constant__ parameter
  __device__ __forceinline__ HestonThetaPath(const Consts& k_) : b(k_.c), k(k_) {}
  __device__ __forceinline__ void load(double x, double v, double q, const TangentState&, long long, long long, bool) {
    b.load(x, v, q);
    dx = dv = dq = 0.0;
  }
  template <bool SAFE>
  __device__ __forceinline__ void step(double z0, double z1) {
    const double v = b.v, sig = sqrt(v), hs = 0.5 / sig;
    b.template step<SAFE>(z0, z1);
    const bool live = b.v > 1e-4;
    const double noise = fma(b.c0, z0, b.c1 * z1);
    const double fx = fma(b.sdt * z0, hs, b.hx);
    const double jac = fma(noise, hs, 1.0 - b.kdt);
    const double drive = fma(sig * noise, k.hdt, k.kappa * (b.theta - v));
    dx = fma(fx, dv, dx) + fma(-0.5, v, sig * z0 * k.hsdt);
    dq = fma(b.dt, dv, dq) + v;
    dv = live ? fma(jac, dv, drive) : 0.0;
  }
  __device__ __forceinline__ bool overflowed() const { return false; }
  __device__ __forceinline__ double sigma() const { return b.sigma(); }
  __device__ __forceinline__ double x() const { return b.x(); }
  __device__ __forceinline__ double q() const { return b.q(); }
  __device__ __forceinline__ double tx(int) const { return dx; }
  __device__ __forceinline__ double tq(int) const { return fma(-k.qshift, q(), dq); }
  __device__ __forceinline__ double tv(int) const { return dv; }
};

// mc_slice_kernel with tangents: same persistent grid-stride loop, same Philox stream (counter = global path id, slice), same
// overflow re-run.  Per-CTA partials [gridDim.x][2 + P]: sum F e^x, count, sum F e^x dx_p over the non-NaN spots.
template <typename TPath, int GAUSS>
__global__ void __launch_bounds__(kSliceThreads, B200SV_SLICE_MINBLOCKS) mc_tangent_slice_kernel(SliceArgs<double> a, TangentState t,
                                                                                                 const __grid_constant__ typename TPath::Consts consts) {
  constexpr int NP = TPath::NP, K = 2 + NP;
  __shared__ double red[K * kSliceThreads / 32];
  exp_table_init();
  if constexpr (GAUSS != kGaussF32) gauss64_table_init();
  double acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.0;
  TPath p(consts);
  const long long stride = (long long)gridDim.x * kSliceThreads;
  for (long long i = (long long)blockIdx.x * kSliceThreads + threadIdx.x; i < a.n; i += stride) {
    double xi = 0.0, vi = a.v_init, qi = 0.0;
    if (!a.init) {
      xi = a.x[i];
      vi = a.v[i];
      qi = a.q[i];
    }
    p.load(xi, vi, qi, t, i, a.n, a.init != 0);
    StepNormals<double, GAUSS> rng(a.seed, a.path_offset + (unsigned long long)i, a.slice);
    run_slice_steps<false, TPath::kPrefetch>(p, rng, a.nsteps);
    if (p.overflowed()) {
      p.load(xi, vi, qi, t, i, a.n, a.init != 0);
      run_slice_steps<true>(p, rng, a.nsteps);
    }
    const double xT = p.x();
    a.x[i] = xT;
    a.v[i] = p.sigma();
    a.q[i] = p.q();
    if constexpr (TPath::kRecordsLastStep) p.record_last_step(i, a.n, xT);
    const double spot = a.forward * exp(xT);
#pragma unroll
    for (int k = 0; k < NP; ++k) {
      const double d = p.tx(k);
      t.dx[k * a.n + i] = d;
      t.dv[k * a.n + i] = p.tv(k);
      t.dq[k * a.n + i] = p.tq(k);
      if (spot == spot) acc[2 + k] = fma(spot, d, acc[2 + k]);
    }
    if (spot == spot) {
      acc[0] += spot;
      acc[1] += 1.0;
    }
  }
  block_sum<K, kSliceThreads>(acc, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) a.partials[K * blockIdx.x + k] = acc[k];
  }
}

// logsv_step_fixed_fast_kernel with the LogSV tangents (DESIGN.md §4.7): the same unit normals W0, W1 [S][n] read from HBM and the same
// clamped primal step (LogsvTangentPath::step<true> calls LogsvPath<double>::step<true> unchanged), so the state it writes back is the fast
// kernel's bit for bit; a.init starts every path at (0, v_init, 0) with the initial tangents.  Per-CTA partials [gridDim.x][2 + P] of
// SpotMoments over the new x: the chain driver keeps the P tangent terms (sum F e^x dx_p) and takes the two re-centring moments from
// spot_moments_impl, as the pricing route does.
__global__ void __launch_bounds__(kThreads, B200SV_SLICE_MINBLOCKS) logsv_tangent_step_fixed_kernel(SliceArgs<double> a, TangentState t,
                                                                                                  const double* __restrict__ W0,
                                                                                                  const double* __restrict__ W1,
                                                                                                  const __grid_constant__ LogsvTangentConsts consts) {
  constexpr int NP = LogsvTangentPath::NP;
  exp_table_init();
  SpotMoments<2 + NP, kThreads> mom;
  LogsvTangentPath p(consts);
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < a.n; i += stride) {
    double xi = 0.0, vi = a.v_init, qi = 0.0;
    if (!a.init) {
      xi = a.x[i];
      vi = a.v[i];
      qi = a.q[i];
    }
    p.load(xi, vi, qi, t, i, a.n, a.init != 0);
    for (int s = 0; s < a.nsteps; ++s) p.step<true>(__ldg(W0 + (size_t)s * a.n + i), __ldg(W1 + (size_t)s * a.n + i));
    const double xT = p.x();
    a.x[i] = xT;
    a.v[i] = p.sigma();
    a.q[i] = p.q();
    const double spot = a.forward * exp(xT);
#pragma unroll
    for (int k = 0; k < NP; ++k) {
      const double d = p.tx(k);
      t.dx[k * a.n + i] = d;
      t.dv[k * a.n + i] = p.tv(k);
      t.dq[k * a.n + i] = p.tq(k);
      mom.add_term(spot, k, d);
    }
    mom.add(spot);
  }
  mom.store(a.partials);
}

// Per-strike sums of the payoff and of its pathwise derivatives.  U = re-centred spot S (LOG_RETURN) or q/ttm (Q_VAR);
// dS_p = F e^x dx_p - mean(F e^x dx_p) over the nanmean's set, dS/dF = S/F; dU_p = dq_p/ttm, dU/dF = 0 under Q_VAR.
// pay = h(U) (C/P) or h(U)/S (IC/IP) with h = (U-K)^+ or (K-U)^+; g = h'(U) dU or (h'(U) dU - pay dS)/S.  A path whose payoff is NaN
// is skipped for every sum.  Row layout per strike: (sum pay, sum pay^2, count, then (sum g, sum g^2) for delta and every parameter).
// SCORE (the Hawkes route, DESIGN.md §3.11): every parameter row also carries the likelihood-ratio term pay * score_p, score [NP][n].
constexpr int kGreeksStrikeChunk = 2;
template <int NP, bool SCORE>
__device__ __forceinline__ void payoff_greeks_body(const double* __restrict__ x, const double* __restrict__ q, const double* __restrict__ dx,
                                                   const double* __restrict__ dq, const double* __restrict__ score, long long n, double ttm,
                                                   double forward, const double* __restrict__ strikes, const int8_t* __restrict__ types, int J,
                                                   int variable_type, const double* __restrict__ moments, double* __restrict__ partials,
                                                   int Kpad) {
  constexpr int KV = 3 + 2 * (1 + NP), KC = KV * kGreeksStrikeChunk;
  __shared__ double red[KC * kThreads / 32];
  __shared__ double sh_mom[2 + NP];
  if (threadIdx.x < 2 + NP) sh_mom[threadIdx.x] = moments[threadIdx.x];
  __syncthreads();
  const double corr = sh_mom[0] / sh_mom[1] - forward;
  double mean_d[NP];
#pragma unroll
  for (int k = 0; k < NP; ++k) mean_d[k] = sh_mom[2 + k] / sh_mom[1];
  const int j0 = blockIdx.y * kGreeksStrikeChunk;
  double kk[kGreeksStrikeChunk];
  int ty[kGreeksStrikeChunk];
  load_strike_chunk(strikes, types, J, j0, kk, ty);
  const bool is_qvar = variable_type == B200SV_Q_VAR;
  const double inv_f = 1.0 / forward, inv_ttm = 1.0 / ttm;
  double acc[KC];
#pragma unroll
  for (int c = 0; c < KC; ++c) acc[c] = 0.0;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    const double fe = forward * exp(x[i]);
    const double spot = fe - corr;
    double dS[1 + NP], dU[1 + NP];
    dS[0] = spot * inv_f;
    dU[0] = is_qvar ? 0.0 : dS[0];
#pragma unroll
    for (int k = 0; k < NP; ++k) {
      dS[1 + k] = fma(fe, dx[k * n + i], -mean_d[k]);
      dU[1 + k] = is_qvar ? dq[k * n + i] * inv_ttm : dS[1 + k];
    }
    const double under = is_qvar ? q[i] * inv_ttm : spot;
    double sc[SCORE ? NP : 1];
    if constexpr (SCORE) {
#pragma unroll
      for (int k = 0; k < NP; ++k) sc[k] = score[k * n + i];
    }
#pragma unroll
    for (int c = 0; c < kGreeksStrikeChunk; ++c) {
      if (ty[c] < 0) continue;
      const bool is_put = ty[c] & 1, inverse = ty[c] >= 2;
      const bool itm = is_put ? under < kk[c] : under > kk[c];
      const double h = itm ? (is_put ? kk[c] - under : under - kk[c]) : 0.0;
      const double hp = itm ? (is_put ? -1.0 : 1.0) : 0.0;
      const double pay = inverse ? h / spot : h;
      if (pay != pay) continue;
      double* a = acc + KV * c;
      a[0] += pay;
      a[1] += pay * pay;
      a[2] += 1.0;
#pragma unroll
      for (int k = 0; k < 1 + NP; ++k) {
        double g = itm ? hp * dU[k] : 0.0;
        if (inverse) g = (g - pay * dS[k]) / spot;
        if constexpr (SCORE) {
          if (k > 0) g = fma(pay, sc[k - 1], g);
        }
        a[3 + 2 * k] += g;
        a[4 + 2 * k] = fma(g, g, a[4 + 2 * k]);
      }
    }
  }
  block_sum<KC, kThreads>(acc, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int c = 0; c < KC; ++c) partials[(size_t)blockIdx.x * Kpad + KV * j0 + c] = acc[c];
  }
}
template <int NP>
__global__ void __launch_bounds__(kThreads) payoff_greeks_kernel(const double* __restrict__ x, const double* __restrict__ q,
                                                                const double* __restrict__ dx, const double* __restrict__ dq, long long n,
                                                                double ttm, double forward, const double* __restrict__ strikes,
                                                                const int8_t* __restrict__ types, int J, int variable_type,
                                                                const double* __restrict__ moments, double* __restrict__ partials, int Kpad) {
  payoff_greeks_body<NP, false>(x, q, dx, dq, nullptr, n, ttm, forward, strikes, types, J, variable_type, moments, partials, Kpad);
}
template <int NP>
__global__ void __launch_bounds__(kThreads) payoff_score_greeks_kernel(const double* __restrict__ x, const double* __restrict__ dx,
                                                                      const double* __restrict__ score, long long n, double ttm, double forward,
                                                                      const double* __restrict__ strikes, const int8_t* __restrict__ types, int J,
                                                                      const double* __restrict__ moments, double* __restrict__ partials, int Kpad) {
  payoff_greeks_body<NP, true>(x, x, dx, dx, score, n, ttm, forward, strikes, types, J, B200SV_LOG_RETURN, moments, partials, Kpad);
}

// prices / std errors exactly as payoff_finalize_kernel (std / sqrt(price_paths)), plus greeks_out[k][Jtot] = df * mean(g_k),
// greeks_se = df * std(g_k) / sqrt(total_paths).  The rough-vol route passes price_paths = 1 (its prices carry the plain std).
__global__ void greeks_finalize_kernel(const double* __restrict__ sums, int KV, int J, int Jtot, double discfactor, double price_paths,
                                       double total_paths, double* __restrict__ prices, double* __restrict__ stderrs, double* __restrict__ greeks,
                                       double* __restrict__ greeks_se) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= J) return;
  const double* s = sums + (size_t)KV * j;
  const double cnt = s[2];
  for (int k = -1; k < (KV - 3) / 2; ++k) {
    const double s1 = k < 0 ? s[0] : s[3 + 2 * k], s2 = k < 0 ? s[1] : s[4 + 2 * k];
    const double mean = s1 / cnt;
    double var = s2 / cnt - mean * mean;
    var = var > 0.0 ? var : 0.0;
    const double m = discfactor * mean, e = discfactor * sqrt(var) / sqrt(k < 0 ? price_paths : total_paths);
    if (k < 0) {
      prices[j] = m;
      stderrs[j] = e;
    } else {
      greeks[(size_t)k * Jtot + j] = m;
      greeks_se[(size_t)k * Jtot + j] = e;
    }
  }
}

// Per-strike (sum g, sum g^2) of the smoothed gamma (DESIGN.md §3.9).  With the other paths held fixed, path i's re-centred spot is
// S_i = (1 - 1/n) F e^{mu_i + s_i Z} - c_i, c_i = (sum_{j != i} Y_j)/n - F = corr - Y_i/n (Y = F e^x, n = the nanmean's count), whose density
// at k is f_i(k) = phi(d) / ((k + c_i) s_i), d = ln((k + c_i) / A_i) / s_i, A_i = (1 - 1/n) F e^{mu_i}, and 0 where k + c_i <= 0.  Per path:
//   LOG_RETURN  C, P: (K/F)^2 f_i(K)     IC: (K/F^2) f_i(K) - 2K/(F^2 S_i) 1{S_i > K}     IP: (K/F^2) f_i(K) + 2K/(F^2 S_i) 1{S_i < K}
//   Q_VAR       C, P: 0                   IC, IP: 2 pay_i / F^2
// A path whose payoff is NaN is skipped, as in the price row.  laststep [2][n] = (s, mu) of mc_tangent_slice_kernel<LastStepPath<.>>.
constexpr int kGammaStrikeChunk = 8;
__global__ void __launch_bounds__(kThreads) payoff_gamma_kernel(const double* __restrict__ x, const double* __restrict__ q,
                                                               const double* __restrict__ laststep, long long n, double ttm, double forward,
                                                               const double* __restrict__ strikes, const int8_t* __restrict__ types, int J,
                                                               int variable_type, const double* __restrict__ moments,
                                                               double* __restrict__ partials, int Kpad) {
  constexpr int KC = 2 * kGammaStrikeChunk;
  __shared__ double red[KC * kThreads / 32];
  __shared__ double sh_mom[2];
  if (threadIdx.x < 2) sh_mom[threadIdx.x] = moments[threadIdx.x];
  __syncthreads();
  const double corr = sh_mom[0] / sh_mom[1] - forward, inv_cnt = 1.0 / sh_mom[1];
  const double log_a0 = log((1.0 - inv_cnt) * forward);       // ln A_i = log_a0 + mu_i
  const int j0 = blockIdx.y * kGammaStrikeChunk;
  double kk[kGammaStrikeChunk];
  int ty[kGammaStrikeChunk];
  load_strike_chunk(strikes, types, J, j0, kk, ty);
  const bool is_qvar = variable_type == B200SV_Q_VAR;
  const double inv_f = 1.0 / forward, inv_f2 = inv_f * inv_f, inv_ttm = 1.0 / ttm;
  constexpr double kInvSqrt2Pi = 0.3989422804014326779;
  double acc[KC];
#pragma unroll
  for (int c = 0; c < KC; ++c) acc[c] = 0.0;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    const double fe = forward * exp(x[i]);
    const double spot = fe - corr;
    const double under = is_qvar ? q[i] * inv_ttm : spot;
    const double s = laststep[i], log_a = log_a0 + laststep[n + i], cshift = fma(-fe, inv_cnt, corr);
#pragma unroll
    for (int c = 0; c < kGammaStrikeChunk; ++c) {
      if (ty[c] < 0) continue;
      const bool is_put = ty[c] & 1, inverse = ty[c] >= 2;
      const bool itm = is_put ? under < kk[c] : under > kk[c];
      const double h = itm ? (is_put ? kk[c] - under : under - kk[c]) : 0.0;
      const double pay = inverse ? h / spot : h;
      if (pay != pay) continue;
      double g;
      if (is_qvar) {
        g = inverse ? 2.0 * pay * inv_f2 : 0.0;
      } else {
        const double kc = kk[c] + cshift;
        double dens = 0.0;
        if (kc > 0.0) {
          const double d = (log(kc) - log_a) / s;
          dens = kInvSqrt2Pi * exp(-0.5 * d * d) / (kc * s);
        }
        g = inverse ? kk[c] * inv_f2 * dens : kk[c] * kk[c] * inv_f2 * dens;
        if (inverse && itm) g += (is_put ? 2.0 : -2.0) * kk[c] * inv_f2 / spot;
      }
      acc[2 * c] += g;
      acc[2 * c + 1] = fma(g, g, acc[2 * c + 1]);
    }
  }
  block_sum<KC, kThreads>(acc, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int c = 0; c < KC; ++c) partials[(size_t)blockIdx.x * Kpad + 2 * j0 + c] = acc[c];
  }
}

// gamma[Jtot] = df * mean(g), gamma_se = df * std(g) / sqrt(total_paths): the sensitivity rows' convention, over the price row's count
// (column 2 of the KV-wide payoff sums: the gamma sums skip the same paths)
__global__ void gamma_finalize_kernel(const double* __restrict__ gsums, const double* __restrict__ sums, int KV, int J, double discfactor,
                                      double total_paths, double* __restrict__ gamma, double* __restrict__ gamma_se) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= J) return;
  const double cnt = sums[(size_t)KV * j + 2];
  const double mean = gsums[2 * j] / cnt;
  double var = gsums[2 * j + 1] / cnt - mean * mean;
  var = var > 0.0 ? var : 0.0;
  gamma[j] = discfactor * mean;
  gamma_se[j] = discfactor * sqrt(var) / sqrt(total_paths);
}

// theta[Jtot] = -df mean(g) / S, theta_se = df std(g) / (S sqrt(total_paths)), g = the d/d dt row of payoff_greeks_kernel<1> over the theta
// pass (column 5, 6 of its KV = 7 sums; the count is column 2, the price row's)
__global__ void theta_finalize_kernel(const double* __restrict__ sums, int J, double discfactor, double nsteps, double total_paths,
                                      double* __restrict__ theta, double* __restrict__ theta_se) {
  constexpr int KV = 3 + 2 * 2;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= J) return;
  const double* s = sums + (size_t)KV * j;
  const double cnt = s[2];
  const double mean = s[5] / cnt;
  double var = s[6] / cnt - mean * mean;
  var = var > 0.0 ? var : 0.0;
  theta[j] = -discfactor * mean / nsteps;
  theta_se[j] = discfactor * sqrt(var) / (nsteps * sqrt(total_paths));
}

// --------------------------------------------------------------------------------------------------------------------
// debug / parity export of the normals the fused kernel draws
// --------------------------------------------------------------------------------------------------------------------
template <int GAUSS>
__global__ void device_normals_kernel(unsigned long long seed, unsigned long long path0, long long n, unsigned int slice,
                                      int nsteps, double* __restrict__ z0, double* __restrict__ z1) {
  if constexpr (GAUSS != kGaussF32) gauss64_table_init();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  StepNormals<double, GAUSS> rng(seed, path0 + (unsigned long long)i, slice);
  if constexpr (GAUSS == kGaussF64) {
    for (int s = 0; s < nsteps; ++s) {
      double a, b;
      rng.get((uint32_t)s, a, b);
      z0[(size_t)s * n + i] = a;
      z1[(size_t)s * n + i] = b;
    }
  } else {
    for (int c = 0; 2 * c < nsteps; ++c) {
      double a0, a1, b0, b1;
      rng.get2((uint32_t)c, a0, a1, b0, b1);
      z0[(size_t)(2 * c) * n + i] = a0;
      z1[(size_t)(2 * c) * n + i] = a1;
      if (2 * c + 1 < nsteps) {
        z0[(size_t)(2 * c + 1) * n + i] = b0;
        z1[(size_t)(2 * c + 1) * n + i] = b1;
      }
    }
  }
}

// exp_pair self-test kernel (tests): out[2i] = exp(L), out[2i+1] = exp(-L)
__global__ void exp_pair_kernel(const double* __restrict__ L, long long n, double* __restrict__ out) {
  exp_table_init();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double a, b;
  exp_pair(L[i], a, b);
  out[2 * i] = a;
  out[2 * i + 1] = b;
}

// the stepper's variant on table units: out[2i] = exp(Ls ln2/256), out[2i+1] = exp(-Ls ln2/256), |Ls| clamped like the stepper does
__global__ void exp_pair_scaled_kernel(const double* __restrict__ Ls, long long n, double* __restrict__ out) {
  exp_table_init();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double a, b;
  exp_pair_scaled(clamp_log_scaled(Ls[i]), a, b);
  out[2 * i] = a;
  out[2 * i + 1] = b;
}

// Box-Muller self-test kernel (tests): the draw functions of philox.cuh / gauss64.cuh on caller-chosen Philox output words, tables
// initialised as the production kernels do.  out[4i..4i+3]: fp64 mode (z0, z1, NaN, NaN); the two-pair modes (z0, z1) of (r0, r1), then of (r2, r3)
template <int GAUSS>
__global__ void box_muller_words_kernel(const uint4* __restrict__ words, long long n, double* __restrict__ out) {
  if constexpr (GAUSS != kGaussF32) gauss64_table_init();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint4 r = words[i];
  double z[4];
  if constexpr (GAUSS == kGaussF64) {
    box_muller_f64_fast(r, z[0], z[1]);
    z[2] = z[3] = __longlong_as_double(0x7ff8000000000000ll);
  } else if constexpr (GAUSS == kGaussF64Paired) {
    box_muller_f64_u32(r.x, r.y, z[0], z[1]);
    box_muller_f64_u32(r.z, r.w, z[2], z[3]);
  } else {
    float a, b, c, d;
    box_muller_f32(r.x, r.y, a, b);
    box_muller_f32(r.z, r.w, c, d);
    z[0] = a;
    z[1] = b;
    z[2] = c;
    z[3] = d;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) out[4 * i + k] = z[k];
}

// fp64 helper self-test kernel (tests): out[i] = op(a[i], b[i]) for the B200SV_DEBUG_* codes of b200sv.h
__global__ void fastmath_kernel(int op, const double* __restrict__ a, const double* __restrict__ b, long long n, double* __restrict__ out) {
  exp_table_init();
  gauss64_table_init();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = a[i];
  double y;
  switch (op) {
    case B200SV_DEBUG_FAST_DIV: y = fast_div(x, b[i]); break;
    case B200SV_DEBUG_FAST_SQRT: y = fast_sqrt(x); break;
    case B200SV_DEBUG_FAST_SQRT_POS: y = fast_sqrt_pos(x); break;
    case B200SV_DEBUG_NEG2_LOG: y = neg2_log((uint32_t)__double2hiint(x), (uint32_t)__double2loint(x)); break;
    default: y = exp_table(x); break;
  }
  out[i] = y;
}

// --------------------------------------------------------------------------------------------------------------------
// host side
// --------------------------------------------------------------------------------------------------------------------
// host-side state of one rank's mailbox (p2p.cuh); created / connected through the b200sv_p2p_* entry points
struct P2pCtx {
  int world, rank, kmax;
  char* mail;                    // own mailbox (cudaMalloc, IPC-exported)
  char* peer[kMaxPeers];         // every rank's mailbox mapped into this process (peer[rank] == mail)
  size_t vals_bytes;             // 2 * world * kmax * 8; flags follow
  unsigned long long published;  // epoch of the last exchange this rank published
  unsigned long long consumed;   // epoch of the last exchange this rank gathered
  double* scratch;               // 1 double (tail of the own mailbox allocation): sink of the protocol-keeping gather below
  unsigned int* status;          // 1 word after scratch: timeout bits set by p2p_gather (p2p.cuh)
  unsigned int spin_limit;
};
static P2pGather make_gather(P2pCtx* c);
__global__ void p2p_gather_kernel(P2pGather g, int K, double* __restrict__ out);
// The double-buffer argument of p2p.cuh needs "publish e+1 only after gathering e" on every rank.  A caller that skips a gather (a
// maturity without strikes, a rank without paths) gets it inserted here: a 1-thread kernel that waits for epoch e's flags.
static P2pPublish make_publish(P2pCtx* c, cudaStream_t st) {
  P2pPublish p{};
  if (!c) return p;
  if (c->consumed < c->published) p2p_gather_kernel<<<1, 32, 0, st>>>(make_gather(c), 1, c->scratch);
  p.world = c->world;
  p.epoch = ++c->published;
  const int slot = (int)(p.epoch & 1ull);
  for (int s = 0; s < c->world; ++s) {
    p.peer_vals[s] = (double*)c->peer[s] + ((size_t)slot * c->world + c->rank) * c->kmax;
    p.peer_flags[s] = (unsigned long long*)(c->peer[s] + c->vals_bytes) + (size_t)slot * c->world + c->rank;
  }
  return p;
}
static P2pGather make_gather(P2pCtx* c) {
  P2pGather g{};
  if (!c) return g;
  g.world = c->world;
  g.kmax = c->kmax;
  g.epoch = c->consumed = c->published;
  g.spin_limit = c->spin_limit;
  g.status = c->status;
  const int slot = (int)(g.epoch & 1ull);
  g.vals = (const double*)c->mail + (size_t)slot * c->world * c->kmax;
  g.flags = (const unsigned long long*)(c->mail + c->vals_bytes) + (size_t)slot * c->world;
  return g;
}

// int(ttm * n) + 1 and dt = linspace(0, ttm, S+1)[1] - [0] (utils/funcs.py:44-47; numpy linspace: step = ttm / S, y[1] = 1*step)
struct StepGrid {
  int S;
  double dt;
};
static StepGrid time_grid(double ttm, int n_per_year) {
  const int S = (int)(ttm * (double)n_per_year) + 1;
  return {S, (S == 1) ? ttm : ttm / (double)S};   // linspace sets the LAST point to `stop` exactly; with S == 1 y[1] is that point
}
// the slice of maturity m of a chain: from ttms[m - 1] (0 for the first) to ttms[m]
static StepGrid maturity_grid(const double* ttms, int m, int n_per_year) { return time_grid(ttms[m] - (m > 0 ? ttms[m - 1] : 0.0), n_per_year); }

// B200SV_GAUSS_* bits -> GaussMode (philox.cuh); -1 = contradictory
static int gauss_mode(int flags) {
  const bool g64 = flags & B200SV_GAUSS_F64, paired = flags & B200SV_GAUSS_F64_PAIRED;
  if (g64 && paired) return -1;
  return paired ? kGaussF64Paired : (g64 ? kGaussF64 : kGaussF32);
}

// ---- model dispatch ------------------------------------------------------------------------------------------------------
// The parameter type picks the model and its consts; the consts type picks the kernel instantiation (HestonConsts::qe the scheme).
static LogsvConsts slice_consts(const b200sv_logsv_params& p, double eta, bool spot, double dt, int) { return make_logsv_consts(p, eta, spot, dt); }
static HestonConsts slice_consts(const b200sv_heston_params& p, double, bool, double dt, int scheme) { return make_heston_consts(p, dt, scheme); }
static LogsvTangentConsts tangent_consts(const b200sv_logsv_params& p, double eta, bool spot, double dt) {
  return make_logsv_tangent_consts(p, eta, spot, dt);
}
static HestonTangentConsts tangent_consts(const b200sv_heston_params& p, double, bool, double dt) { return make_heston_tangent_consts(p, dt); }
static double v_init(const b200sv_logsv_params& p) { return p.sigma0; }
static double v_init(const b200sv_heston_params& p) { return p.v0; }
static LogsvThetaConsts theta_consts(const b200sv_logsv_params& p, double eta, bool spot, double dt, double qshift) {
  return make_logsv_theta_consts(p, eta, spot, dt, qshift);
}
static HestonThetaConsts theta_consts(const b200sv_heston_params& p, double, bool, double dt, double qshift) {
  return make_heston_theta_consts(p, dt, qshift);
}
template <typename TConsts>
using TangentPathOf = std::conditional_t<std::is_same<TConsts, LogsvTangentConsts>::value, LogsvTangentPath, HestonTangentPath>;
template <typename TConsts>
using ThetaPathOf = std::conditional_t<std::is_same<TConsts, LogsvThetaConsts>::value, LogsvThetaPath, HestonThetaPath>;

// (model, Heston scheme, state precision Real, Gaussian mode g) -> mc_slice_kernel; nullptr: the paired check mode on fp32 state
template <typename Real, typename Consts>
using SliceKernel = void (*)(SliceArgs<Real>, Consts);
template <typename Real, typename Path, typename Consts>
static SliceKernel<Real, Consts> slice_kernel_g(int g) {
  if (g == kGaussF32) return mc_slice_kernel<Path, Consts, Real, kGaussF32>;
  if (g == kGaussF64) return mc_slice_kernel<Path, Consts, Real, kGaussF64>;
  if constexpr (std::is_same<Real, double>::value) return mc_slice_kernel<Path, Consts, Real, kGaussF64Paired>;
  return nullptr;
}
template <typename Real>
static SliceKernel<Real, LogsvConsts> slice_kernel(const LogsvConsts&, int g) { return slice_kernel_g<Real, LogsvPath<Real>, LogsvConsts>(g); }
template <typename Real>
static SliceKernel<Real, HestonConsts> slice_kernel(const HestonConsts& c, int g) {
  return c.qe ? slice_kernel_g<Real, HestonPath<Real, true>, HestonConsts>(g) : slice_kernel_g<Real, HestonPath<Real, false>, HestonConsts>(g);
}

// (model, Heston scheme, Gaussian mode fp32 | fp64) -> mc_chain_coop_kernel (fp64 state)
template <typename Consts>
using CoopKernel = void (*)(CoopArgs, const CoopSliceSpec<Consts>*);
template <typename Path, typename Consts>
static CoopKernel<Consts> coop_kernel_g(int g) {
  return g == kGaussF64 ? mc_chain_coop_kernel<Path, Consts, kGaussF64> : mc_chain_coop_kernel<Path, Consts, kGaussF32>;
}
static CoopKernel<LogsvConsts> coop_kernel(const LogsvConsts&, int g) { return coop_kernel_g<LogsvPath<double>, LogsvConsts>(g); }
static CoopKernel<HestonConsts> coop_kernel(const HestonConsts& c, int g) {
  return c.qe ? coop_kernel_g<HestonPath<double, true>, HestonConsts>(g) : coop_kernel_g<HestonPath<double, false>, HestonConsts>(g);
}

// ---- launchers ---------------------------------------------------------------------------------------------------------
// The re-centring moments of a slice: launch(partials) enqueues the slice kernel on `blocks` CTAs, each writing its row of the partials
// [blocks][K] (SpotMoments), then reduce_partials_kernel sums them in fixed order into moments_out[K] and, with a P2P context, publishes
// them to the peers (exchange #1, producer).
template <class Launch>
static int slice_moments(const char* what, int K, int blocks, double* moments_out, cudaStream_t st, P2pCtx* p2p, Launch launch) {
  ensure_pool_threshold();      // device-level callers too: a pool that trims at every synchronisation stalls the whole node (DESIGN.md 5)
  DevBuf partials(st);
  B200SV_CUDA(partials.alloc(sizeof(double) * K * (size_t)blocks));
  launch(partials.as<double>());
  if (int rc = check_launch(what)) return rc;
  reduce_partials_kernel<<<1, 64, 0, st>>>(partials.as<double>(), blocks, K, K, moments_out, make_publish(p2p, st));
  return check_launch("reduce_partials_kernel");
}

// one maturity slice on paths [path_offset, path_offset + n), then their re-centring moments (sum F e^x, count) into moments_out
template <typename Real, typename Consts>
static int launch_slice_k(SliceKernel<Real, Consts> kernel, void* x, void* v, void* q, long long n, long long path_offset, int init,
                          double v_init, int nsteps, int slice_index, double forward, uint64_t seed, const Consts& c, double* moments_out,
                          cudaStream_t st, P2pCtx* p2p) {
  Grid g = persistent_grid(kernel, kSliceThreads, n);
  size_t dyn_smem = 0;
#ifdef B200SV_TUNING   // occupancy sweep for profiles/: cap resident CTAs per SM with dynamic shared memory (tuning builds only)
  if (const char* e = getenv("B200SV_DEBUG_BLOCKS_PER_SM")) {
    const int bps = atoi(e);
    if (bps > 0) {
      dyn_smem = (size_t)(200 * 1024) / bps;
      if constexpr (std::is_same<Consts, LogsvConsts>::value)
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_smem);
      g.blocks = (int)std::min<long long>((long long)device_sm_count() * bps, (n + kSliceThreads - 1) / kSliceThreads);
    }
  }
#endif
  return slice_moments("mc_slice_kernel", 2, g.blocks, moments_out, st, p2p, [&](double* partials) {
    const SliceArgs<Real> a{(Real*)x, (Real*)v, (Real*)q, n, (unsigned long long)path_offset, init, v_init, nsteps, (unsigned int)slice_index,
                            seed, forward, partials};
    kernel<<<g.blocks, g.threads, dyn_smem, st>>>(a, c);
  });
}

template <typename Consts>
static int launch_slice(void* x, void* v, void* q, long long n, long long path_offset, int init, double v_init, int nsteps, int slice_index,
                        double forward, uint64_t seed, int flags, const Consts& c, double* moments_out, cudaStream_t st, P2pCtx* p2p = nullptr) {
  const int g = gauss_mode(flags);
  if (g < 0) return fail(-1, "invalid argument: B200SV_GAUSS_F64 and B200SV_GAUSS_F64_PAIRED are mutually exclusive");
  if (flags & B200SV_STATE_F32) {
    if (const auto k = slice_kernel<float>(c, g))
      return launch_slice_k(k, x, v, q, n, path_offset, init, v_init, nsteps, slice_index, forward, seed, c, moments_out, st, p2p);
  } else if (const auto k = slice_kernel<double>(c, g)) {
    return launch_slice_k(k, x, v, q, n, path_offset, init, v_init, nsteps, slice_index, forward, seed, c, moments_out, st, p2p);
  }
  return fail(-1, "invalid argument: the paired Gaussian check mode needs fp64 state");
}

// kinds: bit 0 = some 'C'/'P', bit 1 = some 'IC'/'IP' in this slice; 0 = unknown (device-level callers) -> general kernel
template <typename Real>
static int launch_payoff_t(const void* x, const void* q, long long n, double ttm, double forward, const double* strikes,
                           const int8_t* types, int J, int variable_type, int kinds, const double* moments, double* sums_out,
                           cudaStream_t st, P2pCtx* p2p = nullptr) {
  if (p2p && 3 * J > p2p->kmax) return fail(-1, "P2P mailbox too small for this slice (max_values < 3*J)");
  const P2pGather gat = make_gather(p2p);      // exchange #1 (consumer): the global re-centring moments
  const int chunks = (J + kStrikeChunk - 1) / kStrikeChunk;
  const int Kpad = 3 * kStrikeChunk * chunks;
  const bool vanilla = kinds == 1;
  Grid g = vanilla ? persistent_grid(payoff_vanilla_kernel<Real>, kThreads, n, kPayoffUnroll) : persistent_grid(payoff_kernel<Real>, kThreads, n);
  g.blocks = std::max(1, g.blocks / chunks);
  ensure_pool_threshold();
  DevBuf partials(st);
  B200SV_CUDA(partials.alloc(sizeof(double) * (size_t)Kpad * g.blocks));
  if (vanilla)
    payoff_vanilla_kernel<Real><<<dim3(g.blocks, chunks), g.threads, 0, st>>>((const Real*)x, (const Real*)q, n, ttm, forward, strikes,
                                                                                types, J, variable_type, moments, partials.as<double>(), Kpad, gat);
  else
    payoff_kernel<Real><<<dim3(g.blocks, chunks), g.threads, 0, st>>>((const Real*)x, (const Real*)q, n, ttm, forward, strikes,
                                                                        types, J, variable_type, moments, partials.as<double>(), Kpad, gat);
  if (int rc = check_launch("payoff_kernel")) return rc;
  reduce_partials_kernel<<<1, 256, 0, st>>>(partials.as<double>(), g.blocks, Kpad, 3 * J, sums_out, make_publish(p2p, st));   // exchange #2 (producer)
  return check_launch("reduce_partials_kernel");
}

static int spot_moments_impl(const double* x, long long n, double forward, double* moments_out, cudaStream_t st, P2pCtx* p2p) {
  const Grid g = persistent_grid(spot_moments_kernel, kThreads, n);
  return slice_moments("spot_moments_kernel", 2, g.blocks, moments_out, st, p2p, [&](double* partials) {
    spot_moments_kernel<<<g.blocks, g.threads, 0, st>>>(x, n, forward, partials);
  });
}

static int payoff_kinds(const int8_t* types, int J) {
  int k = 0;
  for (int j = 0; j < J; ++j) k |= (types[j] >= 2) ? 2 : 1;
  return k;
}

static int validate_chain(int M, const double* ttms, const int* offsets, const double* strikes, const int8_t* types, int variable_type) {
  B200SV_REQUIRE(M >= 1, "M must be >= 1");
  double t0 = 0.0;
  for (int m = 0; m < M; ++m) {
    B200SV_REQUIRE(ttms[m] > t0, "ttms must be positive and strictly increasing");   // data/option_chain.py:147-153
    B200SV_REQUIRE(offsets[m + 1] >= offsets[m], "offsets must be non-decreasing");
    t0 = ttms[m];
  }
  B200SV_REQUIRE(offsets[M] == offsets[0] || (strikes && types), "null pointer");
  for (int j = offsets[0]; j < offsets[M]; ++j)
    if (types[j] < 0 || types[j] > 3) return fail(-3, "unknown option payoff code");      // utils/mc_payoffs.py:83-84
  if (variable_type != B200SV_LOG_RETURN && variable_type != B200SV_Q_VAR)
    return fail(-4, "variable_type not implemented");                                      // utils/mc_payoffs.py:69-70
  return 0;
}

// ---- host-level I/O ------------------------------------------------------------------------------------------------------
// Copies a chain driver's [B][prices | stderrs | ivols][Jalloc] result block into the caller's [B][Jtot] outputs: one device-to-host
// copy, the synchronisation that ends the call, then the scatter on the host (ivols only when ivols_out is given).
static int copy_chain_results(StreamSync& sync, const double* d_out, int B, int Jtot, double* prices_out, double* stderr_out,
                              double* ivols_out, cudaStream_t st) {
  const int Jalloc = std::max(Jtot, 1);
  std::vector<double> h((size_t)3 * Jalloc * B);
  if (Jtot > 0) B200SV_CUDA(cudaMemcpyAsync(h.data(), d_out, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, st));
  if (int rc = sync.done()) return rc;
  for (int b = 0; b < B && Jtot > 0; ++b) {
    const double* o = h.data() + (size_t)3 * Jalloc * b;
    memcpy(prices_out + (size_t)b * Jtot, o, sizeof(double) * Jtot);
    memcpy(stderr_out + (size_t)b * Jtot, o + Jalloc, sizeof(double) * Jtot);
    if (ivols_out) memcpy(ivols_out + (size_t)b * Jtot, o + 2 * Jalloc, sizeof(double) * Jtot);
  }
  return 0;
}

// The chain of a multi-launch chain driver on the device: its strikes and types, the current maturity's re-centring moments and payoff
// sums, and the result block of copy_chain_results for B parameter sets.
struct ChainIO {
  int M, B, Jtot, Jalloc, variable_type;
  const double *ttms, *forwards, *discfactors;
  const int* offsets;
  const int8_t* types;
  cudaStream_t st;
  DevBuf d_strikes, d_types, d_out, d_mom, d_sums;

  ChainIO(int B_, int M_, const double* ttms_, const double* forwards_, const double* discfactors_, const int* offsets_, const int8_t* types_,
          int variable_type_, cudaStream_t s)
      : M(M_), B(B_), Jtot(offsets_[M_] - offsets_[0]), Jalloc(std::max(Jtot, 1)), variable_type(variable_type_), ttms(ttms_),
        forwards(forwards_), discfactors(discfactors_), offsets(offsets_), types(types_), st(s), d_strikes(s), d_types(s), d_out(s), d_mom(s),
        d_sums(s) {}

  // K moments, KV payoff sums per strike and R result rows per parameter set: the pricing layout by default, GreeksChainIO's otherwise
  int upload(const double* strikes, int K = 2, int KV = 3, int R = 3) {
    B200SV_CUDA(d_out.alloc(sizeof(double) * R * Jalloc * B));
    B200SV_CUDA(d_mom.alloc(sizeof(double) * K));
    B200SV_CUDA(d_sums.alloc(sizeof(double) * KV * Jalloc));
    if (Jtot == 0) return 0;
    B200SV_CUDA(d_strikes.upload(strikes + offsets[0], Jtot));
    B200SV_CUDA(d_types.upload(types + offsets[0], Jtot));
    return 0;
  }
  double* moments() const { return d_mom.as<double>(); }

  // maturity m of parameter set b: payoff sums over the state (x, q) -> prices, std errors (/ sqrt(total_paths)) and, with_ivols, implied
  // vols into the result block.  moments_from_x: the re-centring moments are taken from x here, not left by the slice launch.
  int payoff(int b, int m, const void* x, const void* q, bool f32, long long n, double total_paths, bool with_ivols, bool moments_from_x = false) {
    const int J = offsets[m + 1] - offsets[m], jo = offsets[m] - offsets[0];
    if (J == 0) return 0;
    if (moments_from_x)
      if (int rc = spot_moments_impl((const double*)x, n, forwards[m], moments(), st, nullptr)) return rc;
    const double* ks = d_strikes.as<double>() + jo;
    const int8_t* ts = d_types.as<int8_t>() + jo;
    const int kinds = payoff_kinds(types + offsets[m], J);
    if (int rc = f32 ? launch_payoff_t<float>(x, q, n, ttms[m], forwards[m], ks, ts, J, variable_type, kinds, moments(), d_sums.as<double>(), st)
                     : launch_payoff_t<double>(x, q, n, ttms[m], forwards[m], ks, ts, J, variable_type, kinds, moments(), d_sums.as<double>(), st))
      return rc;
    double* o = d_out.as<double>() + (size_t)3 * Jalloc * b + jo;
    const IvolSpec iv{ks, ts, forwards[m], ttms[m], with_ivols ? o + 2 * Jalloc : nullptr};
    payoff_finalize_kernel<<<(J + 127) / 128, 128, 0, st>>>(d_sums.as<double>(), J, discfactors[m], total_paths, o, o + Jalloc, P2pGather{}, iv);
    return check_launch("payoff_finalize_kernel");
  }

  int copy_back(StreamSync& sync, double* prices_out, double* stderr_out, double* ivols_out) const {
    return copy_chain_results(sync, d_out.as<double>(), B, Jtot, prices_out, stderr_out, ivols_out, st);
  }
};

// The chain of a sensitivity driver over nb_path paths and NP parameter directions: ChainIO with the [2 + NP] moments its tangent launch reduces
// into, per-strike sums of the payoff and its sensitivities, their partials (sized once for the widest slice), and the result block
// [prices | std errors | greeks [1 + NP] | greeks_se [1 + NP]][Jalloc].
// SCORE: the payoff launches add the likelihood-ratio term of a score array (payoff_score_greeks_kernel, LOG_RETURN only)
// with_gamma: two more result rows [gamma | gamma_se][Jalloc] after those, filled by payoff_gamma().
// with_theta: two more rows [theta | theta_se][Jalloc] after all of those, filled by payoff_theta() from the theta pass's own moments
// theta_moments() [3] and payoff sums (DESIGN.md §3.12).
template <int NP, bool SCORE = false>
struct GreeksChainIO : ChainIO {
  static constexpr int KV = 3 + 2 * (1 + NP);
  static constexpr int KVT = 3 + 2 * 2;     // payoff_greeks_kernel<1>: price, delta, d/d dt
  long long n;
  bool with_gamma, with_theta;
  Grid gp;      // payoff_greeks_kernel's persistent grid, its blocks split across the strike chunks of a slice
  Grid gg;      // payoff_gamma_kernel's, likewise
  Grid gt;      // payoff_greeks_kernel<1>'s, likewise
  DevBuf d_part, d_gpart, d_gsums, d_tpart, d_tsums, d_tmom;

  GreeksChainIO(int M_, const double* ttms_, const double* forwards_, const double* discfactors_, const int* offsets_, const int8_t* types_,
                int variable_type_, long long nb_path, cudaStream_t s, bool with_gamma_ = false, bool with_theta_ = false)
      : ChainIO(1, M_, ttms_, forwards_, discfactors_, offsets_, types_, variable_type_, s), n(nb_path), with_gamma(with_gamma_),
        with_theta(with_theta_), gp(payoff_grid(nb_path)), gg(with_gamma_ ? persistent_grid(payoff_gamma_kernel, kThreads, nb_path) : Grid{}),
        gt(with_theta_ ? persistent_grid(payoff_greeks_kernel<1>, kThreads, nb_path) : Grid{}), d_part(s), d_gpart(s), d_gsums(s), d_tpart(s),
        d_tsums(s), d_tmom(s) {}

  static Grid payoff_grid(long long nb_path) {
    if constexpr (SCORE) return persistent_grid(payoff_score_greeks_kernel<NP>, kThreads, nb_path);
    else return persistent_grid(payoff_greeks_kernel<NP>, kThreads, nb_path);
  }

  int upload(const double* strikes) {
    int Jmax = 0;
    for (int m = 0; m < M; ++m) Jmax = std::max(Jmax, offsets[m + 1] - offsets[m]);
    const int max_chunks = std::max(1, (Jmax + kGreeksStrikeChunk - 1) / kGreeksStrikeChunk);
    B200SV_CUDA(d_part.alloc(sizeof(double) * (size_t)KV * kGreeksStrikeChunk * max_chunks * gp.blocks));
    if (with_gamma) {
      const int gamma_chunks = std::max(1, (Jmax + kGammaStrikeChunk - 1) / kGammaStrikeChunk);
      B200SV_CUDA(d_gpart.alloc(sizeof(double) * (size_t)2 * kGammaStrikeChunk * gamma_chunks * gg.blocks));
      B200SV_CUDA(d_gsums.alloc(sizeof(double) * 2 * (size_t)Jalloc));
    }
    if (with_theta) {
      B200SV_CUDA(d_tpart.alloc(sizeof(double) * (size_t)KVT * kGreeksStrikeChunk * max_chunks * gt.blocks));
      B200SV_CUDA(d_tsums.alloc(sizeof(double) * KVT * (size_t)Jalloc));
      B200SV_CUDA(d_tmom.alloc(sizeof(double) * 3));
    }
    return ChainIO::upload(strikes, 2 + NP, KV, 2 * (2 + NP) + (with_gamma ? 2 : 0) + (with_theta ? 2 : 0));
  }
  double* theta_moments() const { return d_tmom.as<double>(); }

  // maturity m of S steps: per-strike sums over the state (x, q) and the theta pass's tangents (dx, dq - qshift q) [n] under its moments
  // theta_moments() -> the theta rows of the result block
  int payoff_theta(int m, const double* x, const double* q, const double* dx, const double* dq, int S) {
    const int J = offsets[m + 1] - offsets[m], jo = offsets[m] - offsets[0];
    if (J == 0) return 0;
    const int chunks = (J + kGreeksStrikeChunk - 1) / kGreeksStrikeChunk;
    const int Kpad = KVT * kGreeksStrikeChunk * chunks;
    const int blocks = std::max(1, gt.blocks / chunks);
    payoff_greeks_kernel<1><<<dim3(blocks, chunks), gt.threads, 0, st>>>(x, q, dx, dq, n, ttms[m], forwards[m], d_strikes.as<double>() + jo,
                                                                         d_types.as<int8_t>() + jo, J, variable_type, theta_moments(),
                                                                         d_tpart.as<double>(), Kpad);
    if (int rc = check_launch("payoff_greeks_kernel")) return rc;
    reduce_partials_kernel<<<1, 256, 0, st>>>(d_tpart.as<double>(), blocks, Kpad, KVT * J, d_tsums.as<double>(), P2pPublish{});
    if (int rc = check_launch("reduce_partials_kernel")) return rc;
    double* o = d_out.as<double>() + (size_t)(2 * (2 + NP) + (with_gamma ? 2 : 0)) * Jalloc + jo;
    theta_finalize_kernel<<<(J + 127) / 128, 128, 0, st>>>(d_tsums.as<double>(), J, discfactors[m], (double)S, (double)n, o, o + Jalloc);
    return check_launch("theta_finalize_kernel");
  }

  // maturity m, after payoff(): per-strike sums of the smoothed gamma over the state (x, q) and the last step's laststep [2][n] = (s, mu)
  // -> the gamma rows of the result block, over the count payoff() left in the payoff sums
  int payoff_gamma(int m, const double* x, const double* q, const double* laststep) {
    const int J = offsets[m + 1] - offsets[m], jo = offsets[m] - offsets[0];
    if (J == 0) return 0;
    const int chunks = (J + kGammaStrikeChunk - 1) / kGammaStrikeChunk;
    const int Kpad = 2 * kGammaStrikeChunk * chunks;
    const int blocks = std::max(1, gg.blocks / chunks);
    payoff_gamma_kernel<<<dim3(blocks, chunks), gg.threads, 0, st>>>(x, q, laststep, n, ttms[m], forwards[m], d_strikes.as<double>() + jo,
                                                                     d_types.as<int8_t>() + jo, J, variable_type, moments(), d_gpart.as<double>(),
                                                                     Kpad);
    if (int rc = check_launch("payoff_gamma_kernel")) return rc;
    reduce_partials_kernel<<<1, 256, 0, st>>>(d_gpart.as<double>(), blocks, Kpad, 2 * J, d_gsums.as<double>(), P2pPublish{});
    if (int rc = check_launch("reduce_partials_kernel")) return rc;
    double* o = d_out.as<double>() + (size_t)2 * (2 + NP) * Jalloc + jo;
    gamma_finalize_kernel<<<(J + 127) / 128, 128, 0, st>>>(d_gsums.as<double>(), d_sums.as<double>(), KV, J, discfactors[m], (double)n, o,
                                                           o + Jalloc);
    return check_launch("gamma_finalize_kernel");
  }

  // maturity m: per-strike payoff and sensitivity sums over the state (x, q) and its tangents (dx, dq) [NP][n] -> prices, price-row std
  // errors (/ sqrt(price_paths)) and the 1 + NP sensitivity rows with their standard errors (/ sqrt(n)) into the result block.  SCORE: the
  // rows add the likelihood-ratio term pay * score_p, score [NP][n].
  int payoff(int m, const double* x, const double* q, const double* dx, const double* dq, double price_paths, const double* score = nullptr) {
    const int J = offsets[m + 1] - offsets[m], jo = offsets[m] - offsets[0];
    if (J == 0) return 0;
    const int chunks = (J + kGreeksStrikeChunk - 1) / kGreeksStrikeChunk;
    const int Kpad = KV * kGreeksStrikeChunk * chunks;
    const int blocks = std::max(1, gp.blocks / chunks);
    const double* ks = d_strikes.as<double>() + jo;
    const int8_t* ts = d_types.as<int8_t>() + jo;
    if constexpr (SCORE)
      payoff_score_greeks_kernel<NP><<<dim3(blocks, chunks), gp.threads, 0, st>>>(x, dx, score, n, ttms[m], forwards[m], ks, ts, J, moments(),
                                                                                  d_part.as<double>(), Kpad);
    else
      payoff_greeks_kernel<NP><<<dim3(blocks, chunks), gp.threads, 0, st>>>(x, q, dx, dq, n, ttms[m], forwards[m], ks, ts, J, variable_type,
                                                                            moments(), d_part.as<double>(), Kpad);
    if (int rc = check_launch("payoff_greeks_kernel")) return rc;
    reduce_partials_kernel<<<1, 256, 0, st>>>(d_part.as<double>(), blocks, Kpad, KV * J, d_sums.as<double>(), P2pPublish{});
    if (int rc = check_launch("reduce_partials_kernel")) return rc;
    double* o = d_out.as<double>() + jo;
    greeks_finalize_kernel<<<(J + 127) / 128, 128, 0, st>>>(d_sums.as<double>(), KV, J, Jalloc, discfactors[m], price_paths, (double)n, o,
                                                            o + Jalloc, o + 2 * Jalloc, o + (size_t)(3 + NP) * Jalloc);
    return check_launch("greeks_finalize_kernel");
  }

  // one device-to-host copy of the result block, the synchronisation that ends the call, then the scatter into prices_out, stderr_out [Jtot]
  // and greeks_out, greeks_se_out [1 + NP][Jtot] (a non-empty chain has Jalloc == Jtot, so the block's rows are already the caller's);
  // with_gamma also gamma_out, gamma_se_out [Jtot]
  int copy_back(StreamSync& sync, double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out, double* gamma_out = nullptr,
                double* gamma_se_out = nullptr, double* theta_out = nullptr, double* theta_se_out = nullptr) const {
    const size_t J = (size_t)Jtot, G = (size_t)(1 + NP) * J, T = 2 * J + 2 * G + (with_gamma ? 2 * J : 0);
    std::vector<double> h(T + (with_theta ? 2 * J : 0));
    if (J > 0) B200SV_CUDA(d_out.download(h.data(), h.size()));
    if (int rc = sync.done()) return rc;
    if (J == 0) return 0;
    memcpy(prices_out, h.data(), sizeof(double) * J);
    memcpy(stderr_out, h.data() + J, sizeof(double) * J);
    memcpy(greeks_out, h.data() + 2 * J, sizeof(double) * G);
    memcpy(greeks_se_out, h.data() + 2 * J + G, sizeof(double) * G);
    if (with_gamma) {
      memcpy(gamma_out, h.data() + 2 * J + 2 * G, sizeof(double) * J);
      memcpy(gamma_se_out, h.data() + 3 * J + 2 * G, sizeof(double) * J);
    }
    if (with_theta) {
      memcpy(theta_out, h.data() + T, sizeof(double) * J);
      memcpy(theta_se_out, h.data() + T + J, sizeof(double) * J);
    }
    return 0;
  }

  // the device-level twin of copy_back: the result block's rows copied on the stream into the caller's device arrays prices_out, stderr_out
  // [Jtot] and greeks_out, greeks_se_out [1 + NP][Jtot]; no synchronisation
  int copy_to_device(double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out) const {
    const size_t J = (size_t)Jtot, G = (size_t)(1 + NP) * J;
    if (J == 0) return 0;
    const double* o = d_out.as<double>();
    B200SV_CUDA(cudaMemcpyAsync(prices_out, o, sizeof(double) * J, cudaMemcpyDeviceToDevice, st));
    B200SV_CUDA(cudaMemcpyAsync(stderr_out, o + J, sizeof(double) * J, cudaMemcpyDeviceToDevice, st));
    B200SV_CUDA(cudaMemcpyAsync(greeks_out, o + 2 * J, sizeof(double) * G, cudaMemcpyDeviceToDevice, st));
    B200SV_CUDA(cudaMemcpyAsync(greeks_se_out, o + 2 * J + G, sizeof(double) * G, cudaMemcpyDeviceToDevice, st));
    return 0;
  }
};

// The [3][n] fp64 path state (x, vol, qvar) of a host-level call on the device, or its tangents ([3][NP * n]), and the caller's three arrays
// it is uploaded from (alloc(true)) and copied back to (download).
struct HostState {
  double* h[3];
  size_t n;
  cudaStream_t st;
  DevBuf d;

  HostState(double* x, double* v, double* q, long long n_, cudaStream_t s) : h{x, v, q}, n((size_t)n_), st(s), d(s) {}
  double* dev(int k) const { return d.as<double>() + k * n; }
  int alloc(bool upload) {
    B200SV_CUDA(d.alloc(sizeof(double) * 3 * n));
    for (int k = 0; k < 3 && upload; ++k) B200SV_CUDA(cudaMemcpyAsync(dev(k), h[k], sizeof(double) * n, cudaMemcpyHostToDevice, st));
    return 0;
  }
  int download() const {
    for (int k = 0; k < 3; ++k) B200SV_CUDA(cudaMemcpyAsync(h[k], dev(k), sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    return 0;
  }
};

// ---- host-level chain drivers ----------------------------------------------------------------------------------------------
// Which chain driver?  The cooperative single-launch kernel wins where launch and host overhead matter (small path counts) and loses at
// large ones, where its 128-register budget (slice + payoff phases in one kernel) costs more than 20 launches: it serves
// nb_path <= kCoopMaxPaths.
// B200SV_CHAIN_COOP=0 / 1 forces the multi-launch / cooperative driver (A/B measurements, tests).
constexpr long long kCoopMaxPaths = 4000000;        // LogSV
constexpr long long kCoopMaxPathsHeston = 500000;   // Heston's cheaper step leaves less to hide the fused kernel's register budget behind
static bool use_coop_chain(int flags, long long nb_path, bool heston = false) {
  if (flags & B200SV_STATE_F32) return false;
  const int g = gauss_mode(flags);
  if (g != kGaussF32 && g != kGaussF64) return false;
  static const int mode = [] {
    const char* e = getenv("B200SV_CHAIN_COOP");
    int dev = 0, coop = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    if (!coop) return 0;
    return e ? (e[0] == '0' ? 0 : 2) : 1;      // 0 never, 1 by size, 2 always
  }();
  return mode == 2 || (mode == 1 && nb_path <= (heston ? kCoopMaxPathsHeston : kCoopMaxPaths));
}

// Small-chain fast path: ONE stream-ordered allocation, ONE host-to-device copy (strikes, types and the per-maturity specs of all B sets in
// one blob), ONE cooperative launch per parameter set, ONE device-to-host copy.
template <typename Params>
static int mc_chain_host_coop(const Params* params, int M, const double* ttms, const double* forwards, const double* discfactors,
                              const double* etas, const int* offsets, const double* strikes, const int8_t* types, long long nb_path,
                              int nb_steps_per_year, int is_spot, int variable_type, uint64_t seed, int flags, double* prices_out,
                              double* stderr_out, int scheme, int B, double* ivols_out) {
  using Consts = decltype(slice_consts(*params, 1.0, false, 1.0, scheme));
  using Spec = CoopSliceSpec<Consts>;
  const int Jtot = offsets[M] - offsets[0], Jalloc = std::max(Jtot, 1);
  int Jmax = 1;
  for (int m = 0; m < M; ++m) Jmax = std::max(Jmax, offsets[m + 1] - offsets[m]);
  const int Kpad_max = 3 * kStrikeChunk * ((Jmax + kStrikeChunk - 1) / kStrikeChunk);
  // device arena layout (8-byte units unless noted): [in: strikes Jalloc | specs B*M | types (bytes, padded)] [state 3n] [out B*3*Jalloc] [pm] [pp]
  const size_t spec_bytes = sizeof(Spec) * (size_t)M * B;
  const size_t in_bytes = sizeof(double) * Jalloc + spec_bytes + (((size_t)Jalloc + 7) & ~(size_t)7);
  const size_t out_doubles = (size_t)3 * Jalloc * B;
  std::vector<char> h_in(in_bytes, 0);
  if (Jtot > 0) {
    memcpy(h_in.data(), strikes + offsets[0], sizeof(double) * Jtot);
    memcpy(h_in.data() + sizeof(double) * Jalloc + spec_bytes, types + offsets[0], Jtot);
  }
  Spec* h_specs = (Spec*)(h_in.data() + sizeof(double) * Jalloc);
  for (int b = 0; b < B; ++b) {
    for (int m = 0; m < M; ++m) {
      const auto [S, dt] = maturity_grid(ttms, m, nb_steps_per_year);
      const int J = offsets[m + 1] - offsets[m];
      Spec& sp = h_specs[(size_t)b * M + m];
      sp.c = slice_consts(params[b], etas ? etas[(size_t)b * M + m] : 1.0, is_spot != 0, dt, scheme);
      sp.nsteps = S;
      sp.jo = offsets[m] - offsets[0];
      sp.J = J;
      sp.kinds = J ? payoff_kinds(types + offsets[m], J) : 0;
      sp.forward = forwards[m];
      sp.ttm = ttms[m];
      sp.discfactor = discfactors[m];
    }
  }
  const CoopKernel<Consts> kernel = coop_kernel(h_specs[0].c, gauss_mode(flags));
  const int blocks = persistent_grid(kernel, kSliceThreads, nb_path).blocks;
  const size_t total = in_bytes + sizeof(double) * (3 * (size_t)nb_path + out_doubles + 2 * (size_t)blocks + (size_t)Kpad_max * blocks);
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  DevBuf arena(st);
  B200SV_CUDA(arena.alloc(total));
  B200SV_CUDA(cudaMemcpyAsync(arena.p, h_in.data(), in_bytes, cudaMemcpyHostToDevice, st));      // pageable source: staged before the call returns
  char* base = arena.as<char>();
  const Spec* d_specs = (const Spec*)(base + sizeof(double) * Jalloc);
  double* d_state = (double*)(base + in_bytes);
  double* d_out = d_state + 3 * (size_t)nb_path;
  double* d_pm = d_out + out_doubles;
  for (int b = 0; b < B; ++b) {
    double* out_b = d_out + (size_t)3 * Jalloc * b;
    CoopArgs a{};
    a.x = d_state;
    a.v = d_state + nb_path;
    a.q = d_state + 2 * nb_path;
    a.n = nb_path;
    a.v_init = v_init(params[b]);
    a.seed = seed;
    a.M = M;
    a.variable_type = variable_type;
    a.strikes = (const double*)base;
    a.types = (const int8_t*)(base + sizeof(double) * Jalloc + spec_bytes);
    a.part_mom = d_pm;
    a.part_pay = d_pm + 2 * (size_t)blocks;
    a.Kpad_max = Kpad_max;
    a.total_paths = (double)nb_path;
    a.prices = out_b;
    a.stderrs = out_b + Jalloc;
    a.ivols = ivols_out ? out_b + 2 * Jalloc : nullptr;
    const Spec* sp = d_specs + (size_t)b * M;
    void* kargs[] = {(void*)&a, (void*)&sp};
    if (int rc = check_launch("mc_chain_coop_kernel",
                              cudaLaunchCooperativeKernel((void*)kernel, dim3(blocks), dim3(kSliceThreads), kargs, 0, st)))
      return rc;
  }
  return copy_chain_results(sync, d_out, B, Jtot, prices_out, stderr_out, ivols_out, st);
}

// shared host-level chain driver
template <typename Params>
static int mc_chain_host(const Params* params, int M, const double* ttms, const double* forwards, const double* discfactors, const double* etas,
                         const int* offsets, const double* strikes, const int8_t* types, long long nb_path, int nb_steps_per_year, int is_spot,
                         int variable_type, uint64_t seed, int flags, double* prices_out, double* stderr_out, int scheme = 0, int B = 1,
                         double* ivols_out = nullptr) {
  // B > 1: params points to B parameter sets, etas to [B][M], outputs to [B][Jtot]; the sets run back to back on one stream with the SAME
  // seed (common random numbers => a smooth objective in the parameters), no host synchronisation until the single copy back
  B200SV_REQUIRE(B >= 1, "B must be >= 1");
  B200SV_REQUIRE(nb_path >= 1, "nb_path must be >= 1");
  B200SV_REQUIRE(nb_steps_per_year >= 1, "nb_steps_per_year must be >= 1");
  if (int rc = validate_chain(M, ttms, offsets, strikes, types, variable_type)) return rc;
  if (use_coop_chain(flags, nb_path, std::is_same<Params, b200sv_heston_params>::value))
    return mc_chain_host_coop(params, M, ttms, forwards, discfactors, etas, offsets, strikes, types, nb_path, nb_steps_per_year, is_spot,
                              variable_type, seed, flags, prices_out, stderr_out, scheme, B, ivols_out);
  const bool f32 = flags & B200SV_STATE_F32;
  const size_t esz = f32 ? 4 : 8;
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  DevBuf state(st);
  ChainIO io(B, M, ttms, forwards, discfactors, offsets, types, variable_type, st);
  B200SV_CUDA(state.alloc(3 * esz * (size_t)nb_path));
  if (int rc = io.upload(strikes)) return rc;
  char *x = state.as<char>(), *v = x + esz * (size_t)nb_path, *q = x + 2 * esz * (size_t)nb_path;
  for (int b = 0; b < B; ++b) {
    for (int m = 0; m < M; ++m) {
      const auto [S, dt] = maturity_grid(ttms, m, nb_steps_per_year);
      const auto c = slice_consts(params[b], etas ? etas[(size_t)b * M + m] : 1.0, is_spot != 0, dt, scheme);
      if (int rc = launch_slice(x, v, q, nb_path, 0, m == 0, v_init(params[b]), S, m, forwards[m], seed, flags, c, io.moments(), st)) return rc;
      if (int rc = io.payoff(b, m, x, q, f32, nb_path, (double)nb_path, ivols_out != nullptr)) return rc;
    }
  }
  return io.copy_back(sync, prices_out, stderr_out, ivols_out);
}

template <typename Params>
static int terminal_host(const Params& p, double ttm, long long nb_path, int nb_steps_per_year, int is_spot, double eta, uint64_t seed, int flags,
                         double* x, double* v, double* q, int scheme = 0) {
  B200SV_REQUIRE(nb_path >= 1 && ttm > 0.0 && nb_steps_per_year >= 1, "nb_path, ttm, nb_steps_per_year must be positive");
  B200SV_REQUIRE(!(flags & B200SV_STATE_F32), "terminal values are returned as float64: use B200SV_STATE_F64");
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  HostState s(x, v, q, nb_path, st);
  DevBuf d_mom(st);
  if (int rc = s.alloc(false)) return rc;
  B200SV_CUDA(d_mom.alloc(sizeof(double) * 2));
  const auto [S, dt] = time_grid(ttm, nb_steps_per_year);
  const auto c = slice_consts(p, eta, is_spot != 0, dt, scheme);
  if (int rc = launch_slice(s.dev(0), s.dev(1), s.dev(2), nb_path, 0, 1, v_init(p), S, 0, 1.0, seed, flags, c, d_mom.as<double>(), st)) return rc;
  if (int rc = s.download()) return rc;
  return sync.done();
}

// ---- pathwise sensitivities: host side --------------------------------------------------------------------------------
// fp64 state, Gaussian mode fp32 or fp64 (the two production streams); anything else is an error, not a fallback
static int greeks_gauss(int flags) {
  if (flags & B200SV_STATE_F32) return fail(-1, "invalid argument: pathwise sensitivities need fp64 state (B200SV_STATE_F64)");
  const int g = gauss_mode(flags);
  if (g != kGaussF32 && g != kGaussF64) return fail(-1, "invalid argument: pathwise sensitivities support B200SV_GAUSS_F32 and B200SV_GAUSS_F64");
  return g;
}

// one maturity slice with tangents; moments_out[2 + P] = (sum F e^x, count, sum F e^x dx_p).  laststep != nullptr: the recording variant,
// which also writes (s, mu) of every path's last step to laststep [2][n].  Both variants take the grid of the plain kernel, so the
// moments' reduction order -- and every number the plain kernel produces -- is the same.
template <typename TConsts>
static int launch_tangent_slice(int gauss, double* x, double* v, double* q, const TangentState& t, long long n, long long path_offset, int init,
                                double v_init, int nsteps, int slice_index, double forward, uint64_t seed, const TConsts& c, double* moments_out,
                                cudaStream_t st, double* laststep = nullptr) {
  using TPath = TangentPathOf<TConsts>;
  using RPath = LastStepPath<TPath>;
  const auto kernel = gauss == kGaussF64 ? mc_tangent_slice_kernel<TPath, kGaussF64> : mc_tangent_slice_kernel<TPath, kGaussF32>;
  const Grid g = persistent_grid(kernel, kSliceThreads, n);
  return slice_moments("mc_tangent_slice_kernel", 2 + TPath::NP, g.blocks, moments_out, st, nullptr, [&](double* partials) {
    const SliceArgs<double> a{x, v, q, n, (unsigned long long)path_offset, init, v_init, nsteps, (unsigned int)slice_index, seed, forward, partials};
    if (laststep) {
      const auto rkernel = gauss == kGaussF64 ? mc_tangent_slice_kernel<RPath, kGaussF64> : mc_tangent_slice_kernel<RPath, kGaussF32>;
      rkernel<<<g.blocks, g.threads, 0, st>>>(a, t, LastStepConsts<TPath>{c, laststep});
    } else {
      kernel<<<g.blocks, g.threads, 0, st>>>(a, t, c);
    }
  });
}

// the theta pass of one maturity slice (DESIGN.md §3.12): mc_tangent_slice_kernel<ThetaPathOf<.>> on the same Philox stream and grid shape
// as the tangent pass, its primal the same LogsvPath / HestonPath step; moments_out[3] = (sum F e^x, count, sum F e^x dx_theta)
template <typename HConsts>
static int launch_theta_slice(int gauss, double* x, double* v, double* q, const TangentState& t, long long n, int init, double v_init, int nsteps,
                              int slice_index, double forward, uint64_t seed, const HConsts& c, double* moments_out, cudaStream_t st) {
  using HPath = ThetaPathOf<HConsts>;
  const auto kernel = gauss == kGaussF64 ? mc_tangent_slice_kernel<HPath, kGaussF64> : mc_tangent_slice_kernel<HPath, kGaussF32>;
  const Grid g = persistent_grid(kernel, kSliceThreads, n);
  return slice_moments("mc_tangent_slice_kernel", 2 + HPath::NP, g.blocks, moments_out, st, nullptr, [&](double* partials) {
    const SliceArgs<double> a{x, v, q, n, 0ull, init, v_init, nsteps, (unsigned int)slice_index, seed, forward, partials};
    kernel<<<g.blocks, g.threads, 0, st>>>(a, t, c);
  });
}

// chain driver: per maturity tangent slice -> moments -> per-strike payoff / sensitivity sums -> finalize (stand-alone launches, fixed-order
// reductions).  greeks_out / greeks_se_out: [1 + P][Jtot], row 0 = forward delta.  gamma_out != nullptr: the slices record their last
// step and the smoothed gamma rows gamma_out / gamma_se_out [Jtot] are added (DESIGN.md §3.9), the other outputs unchanged; laststep_out
// [M][2][n_paths_out] (test hook, may be NULL) receives (s, mu) of paths [0, n_paths_out) after every maturity.
// theta_out != nullptr: before each tangent slice a theta pass steps a copy of the state at ttms[m - 1] through the same slice with the
// d/d dt tangent, and theta_out / theta_se_out [Jtot] = -d price / d ttms[m] are added (DESIGN.md §3.12), the other outputs and launches
// unchanged; dtheta_out [M][2][n_paths_out] (test hook, may be NULL) receives (dx, dq) / d dt of paths [0, n_paths_out) after every maturity.
template <typename Params>
static int mc_chain_greeks_host(const Params& p, int M, const double* ttms, const double* forwards, const double* discfactors, const double* etas,
                                const int* offsets, const double* strikes, const int8_t* types, long long nb_path, int nb_steps_per_year,
                                int is_spot, int variable_type, uint64_t seed, int flags, double* prices_out, double* stderr_out,
                                double* greeks_out, double* greeks_se_out, double* gamma_out = nullptr, double* gamma_se_out = nullptr,
                                long long n_paths_out = 0, double* laststep_out = nullptr, double* theta_out = nullptr,
                                double* theta_se_out = nullptr, double* dtheta_out = nullptr) {
  using TConsts = decltype(tangent_consts(p, 1.0, false, 1.0));
  constexpr int NP = TangentPathOf<TConsts>::NP;
  const bool with_gamma = gamma_out != nullptr, with_theta = theta_out != nullptr;
  B200SV_REQUIRE(nb_path >= 1, "nb_path must be >= 1");
  B200SV_REQUIRE(nb_steps_per_year >= 1, "nb_steps_per_year must be >= 1");
  B200SV_REQUIRE(n_paths_out >= 0 && n_paths_out <= nb_path, "n_paths_out must be in [0, nb_path]");
  if (int rc = validate_chain(M, ttms, offsets, strikes, types, variable_type)) return rc;
  const int gauss = greeks_gauss(flags);
  if (gauss < 0) return gauss;
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  const size_t n = (size_t)nb_path, no = laststep_out ? (size_t)n_paths_out : 0, nt = dtheta_out ? (size_t)n_paths_out : 0;
  DevBuf d_state(st);
  GreeksChainIO<NP> io(M, ttms, forwards, discfactors, offsets, types, variable_type, nb_path, st, with_gamma, with_theta);
  B200SV_CUDA(d_state.alloc(sizeof(double) * (3 * n + 3 * (size_t)NP * n + (with_gamma ? 2 * n : 0) + (with_theta ? 6 * n : 0))));
  if (int rc = io.upload(strikes)) return rc;
  double *x = d_state.as<double>(), *v = x + n, *q = v + n;
  const TangentState t{q + n, q + n + NP * n, q + n + 2 * NP * n};
  double* laststep = with_gamma ? q + n + 3 * NP * n : nullptr;     // [2][n], reused across maturities
  double* hstate = q + n + 3 * NP * n + (with_gamma ? 2 * n : 0);     // theta pass: (x, v, q) [3][n], then (dx, dv, dq) [3][n]
  const TangentState ht{hstate + 3 * n, hstate + 4 * n, hstate + 5 * n};
  std::vector<double> h_q(nt * M), qshift(M);                        // the hook's q and S / ttm, to undo tq()'s shift on the host
  for (int m = 0; m < M; ++m) {
    const auto [S, dt] = maturity_grid(ttms, m, nb_steps_per_year);
    const double eta = etas ? etas[m] : 1.0;
    qshift[m] = (double)S / ttms[m];
    if (with_theta) {
      if (m > 0) B200SV_CUDA(cudaMemcpyAsync(hstate, x, sizeof(double) * 3 * n, cudaMemcpyDeviceToDevice, st));   // x, v, q are contiguous
      const auto hc = theta_consts(p, eta, is_spot != 0, dt, qshift[m]);
      if (int rc = launch_theta_slice(gauss, hstate, hstate + n, hstate + 2 * n, ht, nb_path, m == 0, v_init(p), S, m, forwards[m], seed, hc,
                                      io.theta_moments(), st))
        return rc;
    }
    const TConsts c = tangent_consts(p, eta, is_spot != 0, dt);
    if (int rc = launch_tangent_slice(gauss, x, v, q, t, nb_path, 0, m == 0, v_init(p), S, m, forwards[m], seed, c, io.moments(), st, laststep))
      return rc;
    if (int rc = io.payoff(m, x, q, t.dx, t.dq, (double)nb_path)) return rc;
    if (with_gamma) {
      if (int rc = io.payoff_gamma(m, x, q, laststep)) return rc;
      if (no)
        B200SV_CUDA(cudaMemcpy2DAsync(laststep_out + 2 * no * m, sizeof(double) * no, laststep, sizeof(double) * n, sizeof(double) * no, 2,
                                      cudaMemcpyDeviceToHost, st));
    }
    if (!with_theta) continue;
    // the theta rows re-centre with the pricing route's own (sum F e^x, count): the theta pass's primal is the same code on the same
    // normals, and this makes the rows' state and re-centring those of the prices by construction
    B200SV_CUDA(cudaMemcpyAsync(io.theta_moments(), io.moments(), sizeof(double) * 2, cudaMemcpyDeviceToDevice, st));
    if (int rc = io.payoff_theta(m, x, q, ht.dx, ht.dq, S)) return rc;
    if (nt) {
      B200SV_CUDA(cudaMemcpy2DAsync(dtheta_out + 2 * nt * m, sizeof(double) * nt, ht.dx, sizeof(double) * 2 * n, sizeof(double) * nt, 2,
                                    cudaMemcpyDeviceToHost, st));
      B200SV_CUDA(cudaMemcpyAsync(h_q.data() + nt * m, hstate + 2 * n, sizeof(double) * nt, cudaMemcpyDeviceToHost, st));
    }
  }
  if (int rc = io.copy_back(sync, prices_out, stderr_out, greeks_out, greeks_se_out, gamma_out, gamma_se_out, theta_out, theta_se_out)) return rc;
  for (int m = 0; m < M; ++m)
    for (size_t i = 0; i < nt; ++i) dtheta_out[(2 * m + 1) * nt + i] += qshift[m] * h_q[nt * m + i];
  return 0;
}

// chain driver on fixed unit normals resident on the device (DESIGN.md §4.7), per maturity: logsv_tangent_step_fixed_kernel -> its P tangent
// means, the two re-centring moments from spot_moments_impl over x -> per-strike sensitivity sums -> the price and std-error rows from the
// pricing route's own launches (ChainIO::payoff), written over the ones greeks_finalize_kernel left.  So prices and std errors are those of
// b200sv_dev_logsv_step_fixed(fast) + b200sv_dev_spot_moments + b200sv_dev_payoff_sums + b200sv_dev_payoff_finalize on the same normals bit
// for bit, whatever the launch shapes; a maturity without strikes is stepped and not priced, as there.  Asynchronous on `st`.
static int logsv_chain_greeks_fixed(const b200sv_logsv_params& p, int M, const double* ttms, const double* forwards, const double* discfactors,
                                    const double* etas, const int* offsets, const double* strikes, const int8_t* types,
                                    const double* const* W0s, const double* const* W1s, const int* nsteps, const double* dts, long long N,
                                    int is_spot, int variable_type, double* prices_out, double* stderr_out, double* greeks_out,
                                    double* greeks_se_out, cudaStream_t st) {
  constexpr int NP = LogsvTangentPath::NP;
  B200SV_REQUIRE(W0s && W1s && nsteps && dts, "null pointer");
  B200SV_REQUIRE(N >= 1, "N must be >= 1");
  if (int rc = validate_chain(M, ttms, offsets, strikes, types, variable_type)) return rc;
  for (int m = 0; m < M; ++m) {
    B200SV_REQUIRE(W0s[m] && W1s[m], "null pointer");
    B200SV_REQUIRE(nsteps[m] >= 1 && dts[m] > 0.0, "nsteps and dts must be positive");
  }
  B200SV_REQUIRE(offsets[M] == offsets[0] || (prices_out && stderr_out && greeks_out && greeks_se_out), "null pointer");
  ensure_pool_threshold();
  const size_t n = (size_t)N;
  DevBuf d_state(st);
  GreeksChainIO<NP> io(M, ttms, forwards, discfactors, offsets, types, variable_type, N, st);
  B200SV_CUDA(d_state.alloc(sizeof(double) * (3 * n + 3 * (size_t)NP * n)));
  if (int rc = io.upload(strikes)) return rc;
  double *x = d_state.as<double>(), *v = x + n, *q = v + n;
  const TangentState t{q + n, q + n + NP * n, q + n + 2 * NP * n};
  const Grid g = persistent_grid(logsv_tangent_step_fixed_kernel, kThreads, N);
  for (int m = 0; m < M; ++m) {
    const LogsvTangentConsts c = make_logsv_tangent_consts(p, etas ? etas[m] : 1.0, is_spot != 0, dts[m]);
    if (int rc = slice_moments("logsv_tangent_step_fixed_kernel", 2 + NP, g.blocks, io.moments(), st, nullptr, [&](double* partials) {
          const SliceArgs<double> a{x, v, q, N, 0ull, m == 0, p.sigma0, nsteps[m], (unsigned int)m, 0ull, forwards[m], partials};
          logsv_tangent_step_fixed_kernel<<<g.blocks, g.threads, 0, st>>>(a, t, W0s[m], W1s[m], c);
        }))
      return rc;
    if (offsets[m + 1] == offsets[m]) continue;
    if (int rc = spot_moments_impl(x, N, forwards[m], io.moments(), st, nullptr)) return rc;
    if (int rc = io.payoff(m, x, q, t.dx, t.dq, (double)N)) return rc;
    if (int rc = io.ChainIO::payoff(0, m, x, q, false, N, (double)N, false)) return rc;
  }
  return io.copy_to_device(prices_out, stderr_out, greeks_out, greeks_se_out);
}

// one slice from the initial state (0, v_init, 0) with initial tangents, for paths [path_offset, path_offset + n) of Philox slice
// `slice_index`; returns the terminal state and tangents [P][n] (LogSV: dv = d sigma = sigma * d log sigma)
template <typename Params>
static int tangent_terminal_host(const Params& p, double ttm, long long nb_path, int nb_steps_per_year, int is_spot, double eta, uint64_t seed,
                                 int flags, int slice_index, long long path_offset, double* x, double* v, double* q, double* dx, double* dv,
                                 double* dq) {
  using TConsts = decltype(tangent_consts(p, 1.0, false, 1.0));
  constexpr int NP = TangentPathOf<TConsts>::NP;
  B200SV_REQUIRE(nb_path >= 1 && ttm > 0.0 && nb_steps_per_year >= 1, "nb_path, ttm, nb_steps_per_year must be positive");
  B200SV_REQUIRE(slice_index >= 0 && path_offset >= 0, "slice_index and path_offset must be >= 0");
  const int gauss = greeks_gauss(flags);
  if (gauss < 0) return gauss;
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  const size_t n = (size_t)nb_path;
  HostState s(x, v, q, nb_path, st), ds(dx, dv, dq, NP * nb_path, st);
  DevBuf d_mom(st);
  if (int rc = s.alloc(false)) return rc;
  if (int rc = ds.alloc(false)) return rc;
  B200SV_CUDA(d_mom.alloc(sizeof(double) * (2 + NP)));
  const TangentState t{ds.dev(0), ds.dev(1), ds.dev(2)};
  const auto [S, dt] = time_grid(ttm, nb_steps_per_year);
  const TConsts c = tangent_consts(p, eta, is_spot != 0, dt);
  if (int rc = launch_tangent_slice(gauss, s.dev(0), s.dev(1), s.dev(2), t, nb_path, path_offset, 1, v_init(p), S, slice_index, 1.0, seed, c,
                                    d_mom.as<double>(), st))
    return rc;
  if (int rc = s.download()) return rc;
  if (int rc = ds.download()) return rc;
  if (int rc = sync.done()) return rc;
  if (std::is_same<Params, b200sv_logsv_params>::value)
    for (size_t k = 0; k < (size_t)NP; ++k)
      for (size_t i = 0; i < n; ++i) dv[k * n + i] *= v[i];
  return 0;
}

// host-level fixed-random steppers: the state and the normals W0, W1 [S][N] are uploaded, `step` (a device-level stepper) advances the
// state on the device, and the state is copied back in place
template <typename Step>
static int step_fixed_host(double* x, double* v, double* q, const double* W0, const double* W1, int S, long long N, double dt, Step step) {
  B200SV_REQUIRE(x && v && q && (S == 0 || (W0 && W1)), "null pointer");
  B200SV_REQUIRE(S >= 0 && N >= 1 && dt > 0.0, "S, N, dt");
  cudaStream_t st = current_stream();
  StreamSync sync(st);
  HostState s(x, v, q, N, st);
  DevBuf w(st);
  const size_t wb = sizeof(double) * (size_t)N * (size_t)std::max(S, 1);
  if (int rc = s.alloc(true)) return rc;
  B200SV_CUDA(w.alloc(2 * wb));
  if (S > 0) {
    B200SV_CUDA(cudaMemcpyAsync(w.p, W0, wb, cudaMemcpyHostToDevice, st));
    B200SV_CUDA(cudaMemcpyAsync(w.as<double>() + (size_t)N * S, W1, wb, cudaMemcpyHostToDevice, st));
  }
  if (int rc = step(s.dev(0), s.dev(1), s.dev(2), w.as<double>(), w.as<double>() + (size_t)N * S, st)) return rc;
  if (int rc = s.download()) return rc;
  return sync.done();
}

}  // namespace b200sv

#include "rough_kernels.cuh"
#include "hawkes_kernels.cuh"

using namespace b200sv;

extern "C" {

const char* b200sv_last_error(void) { return last_error().c_str(); }
int b200sv_version(void) { return B200SV_VERSION; }
// stream of the calling thread's host-level calls (like cublasSetStream; NULL = the legacy default stream)
int b200sv_set_stream(void* stream) {
  current_stream_ref() = (cudaStream_t)stream;
  return 0;
}
void* b200sv_get_stream(void) { return (void*)current_stream(); }
long long b200sv_launch_count(void) { return launch_count_ref(); }
void b200sv_reset_launch_count(void) { launch_count_ref() = 0; }

int b200sv_logsv_mc_chain(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                          const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                          const int8_t* types, long long nb_path, int nb_steps_per_year, int is_spot_measure, int variable_type,
                          uint64_t seed, int flags, double* prices_out, double* stderr_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out, "null pointer");
  return mc_chain_host(params, M, ttms, forwards, discfactors, etas, offsets, strikes, types, nb_path, nb_steps_per_year, is_spot_measure,
                       variable_type, seed, flags, prices_out, stderr_out);
}

int b200sv_heston_mc_chain(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                           const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                           long long nb_path, int nb_steps_per_year, int variable_type, uint64_t seed, int flags, int scheme,
                           double* prices_out, double* stderr_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out, "null pointer");
  B200SV_REQUIRE(scheme == B200SV_HESTON_EULER_FLOOR || scheme == B200SV_HESTON_QE, "unknown Heston scheme");
  return mc_chain_host(params, M, ttms, forwards, discfactors, nullptr, offsets, strikes, types, nb_path, nb_steps_per_year, 1, variable_type,
                       seed, flags, prices_out, stderr_out, scheme);
}

int b200sv_logsv_mc_chain_batch(const b200sv_logsv_params* params, int B, int M, const double* ttms, const double* forwards,
                                const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                const int8_t* types, long long nb_path, int nb_steps_per_year, int is_spot_measure, uint64_t seed,
                                int flags, double* prices_out, double* stderr_out, double* ivols_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out, "null pointer");
  return mc_chain_host(params, M, ttms, forwards, discfactors, etas, offsets, strikes, types, nb_path, nb_steps_per_year, is_spot_measure,
                       B200SV_LOG_RETURN, seed, flags, prices_out, stderr_out, 0, B, ivols_out);
}

int b200sv_heston_mc_chain_batch(const b200sv_heston_params* params, int B, int M, const double* ttms, const double* forwards,
                                 const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                 long long nb_path, int nb_steps_per_year, uint64_t seed, int flags, int scheme, double* prices_out,
                                 double* stderr_out, double* ivols_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out, "null pointer");
  B200SV_REQUIRE(scheme == B200SV_HESTON_EULER_FLOOR || scheme == B200SV_HESTON_QE, "unknown Heston scheme");
  return mc_chain_host(params, M, ttms, forwards, discfactors, nullptr, offsets, strikes, types, nb_path, nb_steps_per_year, 1, B200SV_LOG_RETURN,
                       seed, flags, prices_out, stderr_out, scheme, B, ivols_out);
}

int b200sv_logsv_mc_chain_greeks(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                 const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                 const int8_t* types, long long nb_path, int nb_steps_per_year, int is_spot_measure, int variable_type,
                                 uint64_t seed, int flags, double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out && greeks_out && greeks_se_out, "null pointer");
  return mc_chain_greeks_host(*params, M, ttms, forwards, discfactors, etas, offsets, strikes, types, nb_path, nb_steps_per_year, is_spot_measure,
                              variable_type, seed, flags, prices_out, stderr_out, greeks_out, greeks_se_out);
}

int b200sv_heston_mc_chain_greeks(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                  const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                  long long nb_path, int nb_steps_per_year, int variable_type, uint64_t seed, int flags, int scheme,
                                  double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out && greeks_out && greeks_se_out, "null pointer");
  B200SV_REQUIRE(scheme == B200SV_HESTON_EULER_FLOOR, "pathwise sensitivities need scheme = B200SV_HESTON_EULER_FLOOR");
  return mc_chain_greeks_host(*params, M, ttms, forwards, discfactors, nullptr, offsets, strikes, types, nb_path, nb_steps_per_year, 1,
                              variable_type, seed, flags, prices_out, stderr_out, greeks_out, greeks_se_out);
}

int b200sv_logsv_mc_chain_greeks_gamma(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                       const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                       const int8_t* types, long long nb_path, int nb_steps_per_year, int is_spot_measure, int variable_type,
                                       uint64_t seed, int flags, double* prices_out, double* stderr_out, double* greeks_out,
                                       double* greeks_se_out, double* gamma_out, double* gamma_se_out, long long n_paths_out,
                                       double* laststep_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out && greeks_out && greeks_se_out && gamma_out &&
                     gamma_se_out,
                 "null pointer");
  return mc_chain_greeks_host(*params, M, ttms, forwards, discfactors, etas, offsets, strikes, types, nb_path, nb_steps_per_year, is_spot_measure,
                              variable_type, seed, flags, prices_out, stderr_out, greeks_out, greeks_se_out, gamma_out, gamma_se_out, n_paths_out,
                              laststep_out);
}

int b200sv_heston_mc_chain_greeks_gamma(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                        const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                        long long nb_path, int nb_steps_per_year, int variable_type, uint64_t seed, int flags, int scheme,
                                        double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out, double* gamma_out,
                                        double* gamma_se_out, long long n_paths_out, double* laststep_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out && greeks_out && greeks_se_out && gamma_out &&
                     gamma_se_out,
                 "null pointer");
  B200SV_REQUIRE(scheme == B200SV_HESTON_EULER_FLOOR, "pathwise sensitivities need scheme = B200SV_HESTON_EULER_FLOOR");
  return mc_chain_greeks_host(*params, M, ttms, forwards, discfactors, nullptr, offsets, strikes, types, nb_path, nb_steps_per_year, 1,
                              variable_type, seed, flags, prices_out, stderr_out, greeks_out, greeks_se_out, gamma_out, gamma_se_out, n_paths_out,
                              laststep_out);
}

int b200sv_logsv_mc_chain_greeks_theta(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                       const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                       const int8_t* types, long long nb_path, int nb_steps_per_year, int is_spot_measure, int variable_type,
                                       uint64_t seed, int flags, double* prices_out, double* stderr_out, double* greeks_out,
                                       double* greeks_se_out, double* gamma_out, double* gamma_se_out, long long n_paths_out,
                                       double* laststep_out, double* theta_out, double* theta_se_out, double* dtheta_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out && greeks_out && greeks_se_out && theta_out &&
                     theta_se_out && (!gamma_out || gamma_se_out),
                 "null pointer");
  return mc_chain_greeks_host(*params, M, ttms, forwards, discfactors, etas, offsets, strikes, types, nb_path, nb_steps_per_year, is_spot_measure,
                              variable_type, seed, flags, prices_out, stderr_out, greeks_out, greeks_se_out, gamma_out, gamma_se_out, n_paths_out,
                              gamma_out ? laststep_out : nullptr, theta_out, theta_se_out, dtheta_out);
}

int b200sv_heston_mc_chain_greeks_theta(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                        const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                        long long nb_path, int nb_steps_per_year, int variable_type, uint64_t seed, int flags, int scheme,
                                        double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out, double* gamma_out,
                                        double* gamma_se_out, long long n_paths_out, double* laststep_out, double* theta_out,
                                        double* theta_se_out, double* dtheta_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out && greeks_out && greeks_se_out && theta_out &&
                     theta_se_out && (!gamma_out || gamma_se_out),
                 "null pointer");
  B200SV_REQUIRE(scheme == B200SV_HESTON_EULER_FLOOR, "pathwise sensitivities need scheme = B200SV_HESTON_EULER_FLOOR");
  return mc_chain_greeks_host(*params, M, ttms, forwards, discfactors, nullptr, offsets, strikes, types, nb_path, nb_steps_per_year, 1,
                              variable_type, seed, flags, prices_out, stderr_out, greeks_out, greeks_se_out, gamma_out, gamma_se_out, n_paths_out,
                              gamma_out ? laststep_out : nullptr, theta_out, theta_se_out, dtheta_out);
}

int b200sv_logsv_tangent_terminal(const b200sv_logsv_params* params, double ttm, long long nb_path, int nb_steps_per_year, int is_spot_measure,
                                  double eta, uint64_t seed, int flags, int slice_index, long long path_offset, double* x, double* sigma,
                                  double* qvar, double* dx, double* dsigma, double* dqvar) {
  B200SV_REQUIRE(params && x && sigma && qvar && dx && dsigma && dqvar, "null pointer");
  return tangent_terminal_host(*params, ttm, nb_path, nb_steps_per_year, is_spot_measure, eta, seed, flags, slice_index, path_offset, x, sigma,
                               qvar, dx, dsigma, dqvar);
}

int b200sv_heston_tangent_terminal(const b200sv_heston_params* params, double ttm, long long nb_path, int nb_steps_per_year, uint64_t seed,
                                   int flags, int slice_index, long long path_offset, double* x, double* var, double* qvar, double* dx,
                                   double* dvar, double* dqvar) {
  B200SV_REQUIRE(params && x && var && qvar && dx && dvar && dqvar, "null pointer");
  return tangent_terminal_host(*params, ttm, nb_path, nb_steps_per_year, 1, 1.0, seed, flags, slice_index, path_offset, x, var, qvar, dx, dvar,
                               dqvar);
}

int b200sv_logsv_terminal(const b200sv_logsv_params* params, double ttm, long long nb_path, int nb_steps_per_year,
                          int is_spot_measure, double eta, uint64_t seed, int flags, double* x, double* sigma, double* qvar) {
  B200SV_REQUIRE(params && x && sigma && qvar, "null pointer");
  return terminal_host(*params, ttm, nb_path, nb_steps_per_year, is_spot_measure, eta, seed, flags, x, sigma, qvar);
}

// simulate_logsv_x_vol_terminal with PER-PATH initial arrays and in-kernel draws (pricers/logsv_pricer.py:1007-1020 accepts length-N x0 / sigma0 /
// qvar0): the three arrays are uploaded, advanced by the fused kernel (init = 0) and copied back in place.  slice_index selects the Philox
// sub-stream (counter word 3), so that successive calls on the same seed continue with fresh normals like the chain pricer's slices.
int b200sv_logsv_terminal_from_state(const b200sv_logsv_params* params, double ttm, long long nb_path, int nb_steps_per_year, int is_spot_measure,
                                     double eta, uint64_t seed, int flags, int slice_index, double* x_inout, double* sigma_inout,
                                     double* qvar_inout) {
  B200SV_REQUIRE(params && x_inout && sigma_inout && qvar_inout, "null pointer");
  B200SV_REQUIRE(nb_path >= 1 && ttm > 0.0 && nb_steps_per_year >= 1 && slice_index >= 0, "nb_path, ttm, nb_steps_per_year must be positive");
  B200SV_REQUIRE(!(flags & B200SV_STATE_F32), "terminal values are returned as float64: use B200SV_STATE_F64");
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  HostState s(x_inout, sigma_inout, qvar_inout, nb_path, st);
  DevBuf d_mom(st);
  if (int rc = s.alloc(true)) return rc;
  B200SV_CUDA(d_mom.alloc(sizeof(double) * 2));
  const auto [S, dt] = time_grid(ttm, nb_steps_per_year);
  const LogsvConsts c = make_logsv_consts(*params, eta, is_spot_measure != 0, dt);
  if (int rc = launch_slice(s.dev(0), s.dev(1), s.dev(2), nb_path, 0, 0, params->sigma0, S, slice_index, 1.0, seed, flags, c, d_mom.as<double>(), st))
    return rc;
  if (int rc = s.download()) return rc;
  return sync.done();
}

int b200sv_heston_terminal(const b200sv_heston_params* params, double ttm, long long nb_path, int nb_steps_per_year,
                           uint64_t seed, int flags, int scheme, double* x, double* var, double* qvar) {
  B200SV_REQUIRE(params && x && var && qvar, "null pointer");
  B200SV_REQUIRE(scheme == B200SV_HESTON_EULER_FLOOR || scheme == B200SV_HESTON_QE, "unknown Heston scheme");
  return terminal_host(*params, ttm, nb_path, nb_steps_per_year, 1, 1.0, seed, flags, x, var, qvar, scheme);
}

// ---- device-level ---------------------------------------------------------------------------------------------------
int b200sv_dev_logsv_slice(void* x, void* sigma, void* qvar, long long n_local, long long path_offset, int init,
                           const b200sv_logsv_params* params, double eta, int is_spot_measure, int nsteps, double dt,
                           int slice_index, double forward, uint64_t seed, int flags, double* moments_out, void* p2p, void* stream) {
  B200SV_REQUIRE(x && sigma && qvar && params && moments_out, "null pointer");
  B200SV_REQUIRE(n_local >= 1 && nsteps >= 1 && dt > 0.0, "n_local, nsteps, dt must be positive");
  const LogsvConsts c = make_logsv_consts(*params, eta, is_spot_measure != 0, dt);
  return launch_slice(x, sigma, qvar, n_local, path_offset, init, params->sigma0, nsteps, slice_index, forward, seed, flags, c, moments_out,
                      (cudaStream_t)stream, (P2pCtx*)p2p);
}

int b200sv_dev_heston_slice(void* x, void* var, void* qvar, long long n_local, long long path_offset, int init,
                            const b200sv_heston_params* params, int nsteps, double dt, int slice_index, double forward,
                            uint64_t seed, int flags, int scheme, double* moments_out, void* p2p, void* stream) {
  B200SV_REQUIRE(x && var && qvar && params && moments_out, "null pointer");
  B200SV_REQUIRE(n_local >= 1 && nsteps >= 1 && dt > 0.0, "n_local, nsteps, dt must be positive");
  B200SV_REQUIRE(scheme == B200SV_HESTON_EULER_FLOOR || scheme == B200SV_HESTON_QE, "unknown Heston scheme");
  const HestonConsts c = make_heston_consts(*params, dt, scheme);
  return launch_slice(x, var, qvar, n_local, path_offset, init, params->v0, nsteps, slice_index, forward, seed, flags, c, moments_out,
                      (cudaStream_t)stream, (P2pCtx*)p2p);
}

int b200sv_dev_payoff_sums(const void* x, const void* qvar, long long n_local, int flags, double ttm, double forward,
                           const double* strikes, const int8_t* types, int J, int variable_type, int payoff_kinds_hint,
                           const double* moments, double* sums_out, void* p2p, void* stream) {
  B200SV_REQUIRE(x && strikes && types && moments && sums_out, "null pointer");
  B200SV_REQUIRE(J >= 1 && n_local >= 1, "J and n_local must be >= 1");
  if (variable_type != B200SV_LOG_RETURN && variable_type != B200SV_Q_VAR) return fail(-4, "variable_type not implemented");
  B200SV_REQUIRE(variable_type == B200SV_LOG_RETURN || qvar, "qvar required for Q_VAR");
  if (flags & B200SV_STATE_F32)
    return launch_payoff_t<float>(x, qvar ? qvar : x, n_local, ttm, forward, strikes, types, J, variable_type, payoff_kinds_hint, moments, sums_out, (cudaStream_t)stream, (P2pCtx*)p2p);
  return launch_payoff_t<double>(x, qvar ? qvar : x, n_local, ttm, forward, strikes, types, J, variable_type, payoff_kinds_hint, moments, sums_out, (cudaStream_t)stream, (P2pCtx*)p2p);
}

int b200sv_dev_payoff_finalize(const double* sums, int J, double discfactor, long long total_paths, double* prices_out,
                               double* stderr_out, void* p2p, void* stream) {
  B200SV_REQUIRE(sums && prices_out && stderr_out && J >= 1, "null pointer / J");
  // exchange #2 (consumer): with a P2P context the global sums are gathered from the mailbox, `sums` holds this rank's local ones
  payoff_finalize_kernel<<<(J + 127) / 128, 128, 0, (cudaStream_t)stream>>>(sums, J, discfactor, (double)total_paths, prices_out, stderr_out,
                                                                            make_gather((P2pCtx*)p2p));
  return check_launch("payoff_finalize_kernel");
}

int b200sv_dev_logsv_step_fixed(double* x, double* sigma, double* qvar, const double* W0, const double* W1, int S, long long N,
                                double dt, const b200sv_logsv_params* params, double eta, int is_spot_measure, int fast, void* stream) {
  B200SV_REQUIRE(x && sigma && qvar && W0 && W1 && params, "null pointer");
  B200SV_REQUIRE(S >= 0 && N >= 1 && dt > 0.0, "S, N, dt");
  if (fast) {
    const LogsvConsts c = make_logsv_consts(*params, eta, is_spot_measure != 0, dt);
    Grid g = persistent_grid(logsv_step_fixed_fast_kernel, kThreads, N);
    logsv_step_fixed_fast_kernel<<<g.blocks, g.threads, 0, (cudaStream_t)stream>>>(x, sigma, qvar, W0, W1, S, N, c);
    return check_launch("logsv_step_fixed_fast_kernel");
  }
  LogsvRaw r{params->theta, params->kappa1, params->kappa2, params->beta, params->volvol, eta,
             is_spot_measure ? -1.0 : 1.0, is_spot_measure ? 0.0 : params->beta * eta, dt};
  Grid g = persistent_grid(logsv_step_fixed_kernel, kThreads, N);
  logsv_step_fixed_kernel<<<g.blocks, g.threads, 0, (cudaStream_t)stream>>>(x, sigma, qvar, W0, W1, S, N, r);
  return check_launch("logsv_step_fixed_kernel");
}

int b200sv_dev_heston_step_fixed(double* x, double* var, double* qvar, const double* W0, const double* W1, int S, long long N,
                                 double dt, const b200sv_heston_params* params, void* stream) {
  B200SV_REQUIRE(x && var && qvar && W0 && W1 && params, "null pointer");
  B200SV_REQUIRE(S >= 0 && N >= 1 && dt > 0.0, "S, N, dt");
  Grid g = persistent_grid(heston_step_fixed_kernel, kThreads, N);
  heston_step_fixed_kernel<<<g.blocks, g.threads, 0, (cudaStream_t)stream>>>(x, var, qvar, W0, W1, S, N, *params, dt);
  return check_launch("heston_step_fixed_kernel");
}

int b200sv_dev_logsv_mc_chain_greeks_fixed(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                           const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                           const int8_t* types, const double* const* W0s, const double* const* W1s, const int* nsteps,
                                           const double* dts, long long N, int is_spot_measure, int variable_type, double* prices_out,
                                           double* stderr_out, double* greeks_out, double* greeks_se_out, void* stream) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets, "null pointer");
  return logsv_chain_greeks_fixed(*params, M, ttms, forwards, discfactors, etas, offsets, strikes, types, W0s, W1s, nsteps, dts, N,
                                  is_spot_measure, variable_type, prices_out, stderr_out, greeks_out, greeks_se_out, (cudaStream_t)stream);
}

int b200sv_dev_spot_moments(const double* x, long long n, double forward, double* moments_out, void* stream) {
  B200SV_REQUIRE(x && moments_out && n >= 1, "null pointer / n");
  return spot_moments_impl(x, n, forward, moments_out, (cudaStream_t)stream, nullptr);
}

// sharded rough-LogSV / Hawkes slices (multi_gpu.py): the steppers of rough_kernels.cuh / hawkes_kernels.cuh on a contiguous range of GLOBAL
// path ids, followed by this rank's re-centring moments (published to the peer-memory mailbox when `p2p` is given) -- the same two
// exchanges per maturity as the LogSV chain
int b200sv_dev_hawkesjd_slice(double* x, double* lambda_p, double* lambda_m, long long n_local, long long path_offset, int init,
                              const b200sv_hawkes_params* params, int nsteps, double dt, int slice_index, double forward, uint64_t seed,
                              int flags, double* moments_out, void* p2p, void* stream) {
  B200SV_REQUIRE(x && lambda_p && lambda_m && params && moments_out, "null pointer");
  B200SV_REQUIRE(n_local >= 1 && nsteps >= 1 && dt > 0.0 && slice_index >= 0, "n_local, nsteps, dt must be positive");
  B200SV_REQUIRE(!(flags & B200SV_STATE_F32), "the Hawkes route is float64 only");
  return launch_hawkes_slice(x, lambda_p, lambda_m, n_local, path_offset, init, *params, nsteps, dt, slice_index, forward, seed, flags,
                             moments_out, (cudaStream_t)stream, (P2pCtx*)p2p);
}

int b200sv_dev_hawkesjd_exact_slice(double* x, double* lambda_p, double* lambda_m, long long n_local, long long path_offset, int init,
                                    const b200sv_hawkes_params* params, double tau, int slice_index, double forward, uint64_t seed,
                                    long long max_candidates, int* overflow, double* moments_out, void* p2p, void* stream) {
  B200SV_REQUIRE(x && lambda_p && lambda_m && params && overflow && moments_out, "null pointer");
  B200SV_REQUIRE(n_local >= 1 && tau > 0.0 && slice_index >= 0, "n_local and tau must be positive");
  return launch_hawkes_exact_slice(x, lambda_p, lambda_m, n_local, path_offset, init, *params, tau, slice_index, forward, seed,
                                   hawkes_exact_budget(max_candidates), overflow, nullptr, 0, moments_out, (cudaStream_t)stream, (P2pCtx*)p2p);
}

int b200sv_dev_rough_logsv_slice(double* log_spot, double* vol_factors, double* qvar, long long n_local, long long path_offset,
                                 const b200sv_logsv_params* params, int n_factors, const double* weights, const double* nodes, int nsteps,
                                 double h, double forward, uint64_t seed, int flags, double* moments_out, void* p2p, void* stream) {
  B200SV_REQUIRE(log_spot && qvar && params && weights && nodes && moments_out, "null pointer");
  B200SV_REQUIRE(n_local >= 1 && nsteps >= 1 && h > 0.0, "n_local, nsteps, h must be positive");
  B200SV_REQUIRE(n_factors >= 1 && n_factors <= kMaxRoughFactors, "1 <= n_factors <= 8");
  B200SV_REQUIRE(!(flags & B200SV_STATE_F32), "the rough-vol route is float64 only");
  const int g = gauss_mode(flags);
  B200SV_REQUIRE(g == kGaussF32 || g == kGaussF64, "gauss flags");
  const RoughConsts c = make_rough_consts(*params, n_factors, weights, nodes, h);
  if (int rc = launch_rough(n_factors, log_spot, vol_factors, qvar, nullptr, nullptr, nsteps, n_local, c, seed, path_offset, g, (cudaStream_t)stream))
    return rc;
  return spot_moments_impl(log_spot, n_local, forward, moments_out, (cudaStream_t)stream, (P2pCtx*)p2p);
}

// ---- host-level fixed-random steppers and payoffs ------------------------------------------------------------------------
int b200sv_logsv_step_fixed(double* x, double* sigma, double* qvar, const double* W0, const double* W1, int S, long long N,
                            double dt, const b200sv_logsv_params* params, double eta, int is_spot_measure) {
  B200SV_REQUIRE(params, "null pointer");
  return step_fixed_host(x, sigma, qvar, W0, W1, S, N, dt, [&](double* dx, double* dv, double* dq, const double* w0, const double* w1, cudaStream_t st) {
    return b200sv_dev_logsv_step_fixed(dx, dv, dq, w0, w1, S, N, dt, params, eta, is_spot_measure, 0, st);
  });
}

int b200sv_heston_step_fixed(double* x, double* var, double* qvar, const double* W0, const double* W1, int S, long long N,
                             double dt, const b200sv_heston_params* params) {
  B200SV_REQUIRE(params, "null pointer");
  return step_fixed_host(x, var, qvar, W0, W1, S, N, dt, [&](double* dx, double* dv, double* dq, const double* w0, const double* w1, cudaStream_t st) {
    return b200sv_dev_heston_step_fixed(dx, dv, dq, w0, w1, S, N, dt, params, st);
  });
}

int b200sv_mc_payoffs(const double* x, const double* qvar, long long N, double ttm, double forward, const double* strikes,
                      const int8_t* types, int J, double discfactor, int variable_type, double* prices_out, double* stderr_out) {
  B200SV_REQUIRE(x && strikes && types && prices_out && stderr_out, "null pointer");
  B200SV_REQUIRE(N >= 1 && J >= 1, "N and J must be >= 1");
  for (int j = 0; j < J; ++j)
    if (types[j] < 0 || types[j] > 3) return fail(-3, "unknown option payoff code");
  if (variable_type != B200SV_LOG_RETURN && variable_type != B200SV_Q_VAR) return fail(-4, "variable_type not implemented");
  B200SV_REQUIRE(variable_type == B200SV_LOG_RETURN || qvar, "qvar required for Q_VAR");
  cudaStream_t st = current_stream();
  StreamSync sync(st);
  DevBuf d(st), dk(st), dt_(st), d_mom(st), d_sums(st), d_out(st);
  const size_t nb = sizeof(double) * (size_t)N;
  B200SV_CUDA(d.alloc(2 * nb));
  B200SV_CUDA(dk.alloc(sizeof(double) * J));
  B200SV_CUDA(dt_.alloc(J));
  B200SV_CUDA(d_mom.alloc(sizeof(double) * 2));
  B200SV_CUDA(d_sums.alloc(sizeof(double) * 3 * J));
  B200SV_CUDA(d_out.alloc(sizeof(double) * 2 * J));
  B200SV_CUDA(cudaMemcpyAsync(d.p, x, nb, cudaMemcpyHostToDevice, st));
  if (qvar) B200SV_CUDA(cudaMemcpyAsync(d.as<double>() + N, qvar, nb, cudaMemcpyHostToDevice, st));
  B200SV_CUDA(cudaMemcpyAsync(dk.p, strikes, sizeof(double) * J, cudaMemcpyHostToDevice, st));
  B200SV_CUDA(cudaMemcpyAsync(dt_.p, types, J, cudaMemcpyHostToDevice, st));
  const double* dx = d.as<double>();
  if (int rc = b200sv_dev_spot_moments(dx, N, forward, d_mom.as<double>(), st)) return rc;
  if (int rc = launch_payoff_t<double>(dx, dx + N, N, ttm, forward, dk.as<double>(), dt_.as<int8_t>(), J, variable_type, payoff_kinds(types, J),
                                       d_mom.as<double>(), d_sums.as<double>(), st))
    return rc;
  if (int rc = b200sv_dev_payoff_finalize(d_sums.as<double>(), J, discfactor, N, d_out.as<double>(), d_out.as<double>() + J, nullptr, st)) return rc;
  B200SV_CUDA(cudaMemcpyAsync(prices_out, d_out.p, sizeof(double) * J, cudaMemcpyDeviceToHost, st));
  B200SV_CUDA(cudaMemcpyAsync(stderr_out, d_out.as<double>() + J, sizeof(double) * J, cudaMemcpyDeviceToHost, st));
  return sync.done();
}

int b200sv_device_normals(uint64_t seed, long long path0, long long n, int slice, int nsteps, int flags, double* z0, double* z1) {
  B200SV_REQUIRE(z0 && z1 && n >= 1 && nsteps >= 1, "null pointer / sizes");
  const int g = gauss_mode(flags);
  B200SV_REQUIRE(g >= 0, "B200SV_GAUSS_F64 and B200SV_GAUSS_F64_PAIRED are mutually exclusive");
  cudaStream_t st = current_stream();
  StreamSync sync(st);
  DevBuf d(st);
  const size_t nb = sizeof(double) * (size_t)n * nsteps;
  B200SV_CUDA(d.alloc(2 * nb));
  double *d0 = d.as<double>(), *d1 = d0 + (size_t)n * nsteps;
  const int blocks = (int)((n + 127) / 128);
  if (g == kGaussF64)
    device_normals_kernel<kGaussF64><<<blocks, 128, 0, st>>>(seed, (unsigned long long)path0, n, (unsigned)slice, nsteps, d0, d1);
  else if (g == kGaussF64Paired)
    device_normals_kernel<kGaussF64Paired><<<blocks, 128, 0, st>>>(seed, (unsigned long long)path0, n, (unsigned)slice, nsteps, d0, d1);
  else
    device_normals_kernel<kGaussF32><<<blocks, 128, 0, st>>>(seed, (unsigned long long)path0, n, (unsigned)slice, nsteps, d0, d1);
  if (int rc = check_launch("device_normals_kernel")) return rc;
  B200SV_CUDA(cudaMemcpyAsync(z0, d0, nb, cudaMemcpyDeviceToHost, st));
  B200SV_CUDA(cudaMemcpyAsync(z1, d1, nb, cudaMemcpyDeviceToHost, st));
  return sync.done();
}

int b200sv_debug_exp_pair_scaled(const double* Ls, long long n, double* out /* 2n */) {
  B200SV_REQUIRE(Ls && out && n >= 1, "null pointer / n");
  cudaStream_t st = current_stream();
  StreamSync sync(st);
  DevBuf dl(st), dout(st);
  B200SV_CUDA(dl.alloc(sizeof(double) * n));
  B200SV_CUDA(dout.alloc(sizeof(double) * 2 * n));
  B200SV_CUDA(cudaMemcpyAsync(dl.p, Ls, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  exp_pair_scaled_kernel<<<(int)((n + 127) / 128), 128, 0, st>>>(dl.as<double>(), n, dout.as<double>());
  if (int rc = check_launch("exp_pair_scaled_kernel")) return rc;
  B200SV_CUDA(cudaMemcpyAsync(out, dout.p, sizeof(double) * 2 * n, cudaMemcpyDeviceToHost, st));
  return sync.done();
}

int b200sv_debug_box_muller(const uint32_t* words, long long n, int flags, double* z_out) {
  B200SV_REQUIRE(words && z_out && n >= 1, "null pointer / n");
  const int g = gauss_mode(flags);
  B200SV_REQUIRE(g >= 0, "B200SV_GAUSS_F64 and B200SV_GAUSS_F64_PAIRED are mutually exclusive");
  cudaStream_t st = current_stream();
  StreamSync sync(st);
  DevBuf dw(st), dout(st);
  B200SV_CUDA(dw.alloc(sizeof(uint4) * n));
  B200SV_CUDA(dout.alloc(sizeof(double) * 4 * n));
  B200SV_CUDA(cudaMemcpyAsync(dw.p, words, sizeof(uint4) * n, cudaMemcpyHostToDevice, st));
  const int blocks = (int)((n + 127) / 128);
  if (g == kGaussF64)
    box_muller_words_kernel<kGaussF64><<<blocks, 128, 0, st>>>(dw.as<uint4>(), n, dout.as<double>());
  else if (g == kGaussF64Paired)
    box_muller_words_kernel<kGaussF64Paired><<<blocks, 128, 0, st>>>(dw.as<uint4>(), n, dout.as<double>());
  else
    box_muller_words_kernel<kGaussF32><<<blocks, 128, 0, st>>>(dw.as<uint4>(), n, dout.as<double>());
  if (int rc = check_launch("box_muller_words_kernel")) return rc;
  B200SV_CUDA(cudaMemcpyAsync(z_out, dout.p, sizeof(double) * 4 * n, cudaMemcpyDeviceToHost, st));
  return sync.done();
}

int b200sv_debug_fastmath(int op, const double* a, const double* b, long long n, double* out) {
  B200SV_REQUIRE(a && out && n >= 1, "null pointer / n");
  B200SV_REQUIRE(op >= B200SV_DEBUG_FAST_DIV && op <= B200SV_DEBUG_EXP_TABLE, "unknown B200SV_DEBUG_* operation");
  B200SV_REQUIRE(op != B200SV_DEBUG_FAST_DIV || b, "fast_div needs the divisors b");
  cudaStream_t st = current_stream();
  StreamSync sync(st);
  DevBuf da(st), db(st), dout(st);
  B200SV_CUDA(da.alloc(sizeof(double) * n));
  B200SV_CUDA(dout.alloc(sizeof(double) * n));
  B200SV_CUDA(cudaMemcpyAsync(da.p, a, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  if (op == B200SV_DEBUG_FAST_DIV) {
    B200SV_CUDA(db.alloc(sizeof(double) * n));
    B200SV_CUDA(cudaMemcpyAsync(db.p, b, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  }
  fastmath_kernel<<<(int)((n + 127) / 128), 128, 0, st>>>(op, da.as<double>(), db.as<double>(), n, dout.as<double>());
  if (int rc = check_launch("fastmath_kernel")) return rc;
  B200SV_CUDA(cudaMemcpyAsync(out, dout.p, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
  return sync.done();
}

int b200sv_debug_hawkes_clocks(const uint32_t* r, const double* lambda, long long n, double dt, const b200sv_hawkes_params* params,
                               double* out) {
  B200SV_REQUIRE(r && lambda && params && out && n >= 1 && dt > 0.0, "null pointer / n / dt");
  cudaStream_t st = current_stream();
  StreamSync sync(st);
  DevBuf dr(st), dl(st), dout(st);
  B200SV_CUDA(dr.alloc(sizeof(uint32_t) * n));
  B200SV_CUDA(dl.alloc(sizeof(double) * n));
  B200SV_CUDA(dout.alloc(sizeof(double) * 6 * n));
  B200SV_CUDA(cudaMemcpyAsync(dr.p, r, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, st));
  B200SV_CUDA(cudaMemcpyAsync(dl.p, lambda, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  hawkes_clocks_kernel<<<(int)((n + 127) / 128), 128, 0, st>>>(dr.as<uint32_t>(), dl.as<double>(), n, make_hawkes_consts(*params, dt),
                                                               dout.as<double>());
  if (int rc = check_launch("hawkes_clocks_kernel")) return rc;
  B200SV_CUDA(cudaMemcpyAsync(out, dout.p, sizeof(double) * 6 * n, cudaMemcpyDeviceToHost, st));
  return sync.done();
}

int b200sv_debug_exp_pair(const double* L, long long n, double* out /* 2n */) {
  B200SV_REQUIRE(L && out && n >= 1, "null pointer / n");
  cudaStream_t st = current_stream();
  StreamSync sync(st);
  DevBuf dl(st), dout(st);
  B200SV_CUDA(dl.alloc(sizeof(double) * n));
  B200SV_CUDA(dout.alloc(sizeof(double) * 2 * n));
  B200SV_CUDA(cudaMemcpyAsync(dl.p, L, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  exp_pair_kernel<<<(int)((n + 127) / 128), 128, 0, st>>>(dl.as<double>(), n, dout.as<double>());
  if (int rc = check_launch("exp_pair_kernel")) return rc;
  B200SV_CUDA(cudaMemcpyAsync(out, dout.p, sizeof(double) * 2 * n, cudaMemcpyDeviceToHost, st));
  return sync.done();
}

int b200sv_logsv_vol_paths(const b200sv_logsv_params* params, double ttm, long long nb_path, int nb_steps_per_year, int is_spot_measure,
                           uint64_t seed, const double* brownians, double* sigma_t_out) {
  B200SV_REQUIRE(params && sigma_t_out, "null pointer");
  B200SV_REQUIRE(nb_path >= 1 && ttm > 0.0 && nb_steps_per_year >= 1, "nb_path, ttm, nb_steps_per_year must be positive");
  const auto [S, dt] = time_grid(ttm, nb_steps_per_year);
  // adj = beta under the inverse measure, no eta (pricers/logsv_pricer.py:929-932)
  LogsvRaw r{params->theta, params->kappa1, params->kappa2, params->beta, params->volvol, 1.0, is_spot_measure ? -1.0 : 1.0,
             is_spot_measure ? 0.0 : params->beta, dt};
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  DevBuf d_out(st), d_w(st);
  const size_t ob = sizeof(double) * (size_t)(S + 1) * (size_t)nb_path, wb = sizeof(double) * (size_t)S * (size_t)nb_path;
  B200SV_CUDA(d_out.alloc(ob));
  if (brownians) {
    B200SV_CUDA(d_w.alloc(wb));
    B200SV_CUDA(cudaMemcpyAsync(d_w.p, brownians, wb, cudaMemcpyHostToDevice, st));
  }
  Grid g = persistent_grid(logsv_vol_paths_kernel, kThreads, nb_path);
  logsv_vol_paths_kernel<<<g.blocks, g.threads, 0, st>>>(d_out.as<double>(), d_w.as<double>(), S, nb_path, r, params->sigma0, seed, 0ull);
  if (int rc = check_launch("logsv_vol_paths_kernel")) return rc;
  B200SV_CUDA(cudaMemcpyAsync(sigma_t_out, d_out.p, ob, cudaMemcpyDeviceToHost, st));
  return sync.done();
}

// ---- rough-LogSV multi-factor MC (rough_kernels.cuh) ------------------------------------------------------------------------
int b200sv_rough_logsv_mc_chain(const b200sv_logsv_params* params, int B, int n_factors, const double* weights, const double* nodes, int M,
                                const double* ttms, const double* forwards, const double* discfactors, const int* offsets, const double* strikes,
                                const int8_t* types, long long nb_path, const int* nsteps, const double* hs, const double* Z0, const double* Z1,
                                long long z_rows, int variable_type, uint64_t seed, int flags, double* prices_out, double* stderr_out,
                                double* ivols_out, double* states_out) {
  B200SV_REQUIRE(params && weights && nodes && ttms && forwards && discfactors && offsets && nsteps && hs && prices_out && stderr_out, "null pointer");
  return rough_chain_host(params, B, n_factors, weights, nodes, M, ttms, forwards, discfactors, offsets, strikes, types, nb_path, nsteps, hs, Z0, Z1,
                          z_rows, variable_type, seed, flags, prices_out, stderr_out, ivols_out, states_out);
}

int b200sv_rough_logsv_mc_chain_greeks(const b200sv_logsv_params* params, int n_factors, const double* weights, const double* nodes, int M,
                                       const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                       const double* strikes, const int8_t* types, long long nb_path, const int* nsteps, const double* hs,
                                       const double* Z0, const double* Z1, long long z_rows, int variable_type, uint64_t seed, int flags,
                                       double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out, double* states_out,
                                       double* tangents_out, double* resets_out) {
  B200SV_REQUIRE(params && weights && nodes && ttms && forwards && discfactors && offsets && nsteps && hs && prices_out && stderr_out && greeks_out &&
                     greeks_se_out,
                 "null pointer");
  return rough_chain_greeks_host(*params, n_factors, weights, nodes, M, ttms, forwards, discfactors, offsets, strikes, types, nb_path, nsteps, hs, Z0,
                                 Z1, z_rows, variable_type, seed, flags, prices_out, stderr_out, greeks_out, greeks_se_out, states_out, tangents_out,
                                 resets_out);
}

int b200sv_rough_logsv_mc_chain_greeks_theta(const b200sv_logsv_params* params, int n_factors, const double* weights, const double* nodes, int M,
                                             const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                             const double* strikes, const int8_t* types, long long nb_path, const int* nsteps, const double* hs,
                                             const double* Z0, const double* Z1, long long z_rows, int variable_type, uint64_t seed, int flags,
                                             double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out, double* states_out,
                                             double* tangents_out, double* resets_out, double* theta_out, double* theta_se_out,
                                             long long n_paths_out, double* dtheta_out) {
  B200SV_REQUIRE(params && weights && nodes && ttms && forwards && discfactors && offsets && nsteps && hs && prices_out && stderr_out && greeks_out &&
                     greeks_se_out && theta_out && theta_se_out,
                 "null pointer");
  return rough_chain_greeks_host(*params, n_factors, weights, nodes, M, ttms, forwards, discfactors, offsets, strikes, types, nb_path, nsteps, hs, Z0,
                                 Z1, z_rows, variable_type, seed, flags, prices_out, stderr_out, greeks_out, greeks_se_out, states_out, tangents_out,
                                 resets_out, theta_out, theta_se_out, n_paths_out, dtheta_out);
}

// ---- Hawkes jump-diffusion MC (hawkes_kernels.cuh) ---------------------------------------------------------------------------
int b200sv_hawkesjd_mc_chain(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards, const double* discfactors,
                             const int* offsets, const double* strikes, const int8_t* types, long long nb_path, int variable_type, uint64_t seed,
                             int flags, double* prices_out, double* stderr_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out, "null pointer");
  return hawkes_chain_host(params, M, ttms, forwards, discfactors, offsets, strikes, types, nb_path, variable_type, seed, flags, prices_out,
                           stderr_out);
}

int b200sv_hawkesjd_mc_chain_greeks(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                    const double* discfactors, const int* offsets, const double* strikes, const int8_t* types, long long nb_path,
                                    int variable_type, uint64_t seed, int flags, double* prices_out, double* stderr_out, double* greeks_out,
                                    double* greeks_se_out, long long n_paths_out, double* states_out, double* tangents_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out && greeks_out && greeks_se_out, "null pointer");
  return hawkes_chain_greeks_host(params, M, ttms, forwards, discfactors, offsets, strikes, types, nb_path, variable_type, seed, flags,
                                  prices_out, stderr_out, greeks_out, greeks_se_out, n_paths_out, states_out, tangents_out);
}

int b200sv_hawkesjd_terminal(const b200sv_hawkes_params* params, double ttm, long long nb_path, uint64_t seed, int flags, int slice_index,
                             int use_initial_arrays, double* x_inout, double* lambda_p_inout, double* lambda_m_inout) {
  B200SV_REQUIRE(params && x_inout && lambda_p_inout && lambda_m_inout, "null pointer");
  B200SV_REQUIRE(nb_path >= 1 && ttm > 0.0 && slice_index >= 0, "nb_path, ttm must be positive");
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  HostState s(x_inout, lambda_p_inout, lambda_m_inout, nb_path, st);
  DevBuf d_mom(st);
  if (int rc = s.alloc(use_initial_arrays != 0)) return rc;
  B200SV_CUDA(d_mom.alloc(sizeof(double) * 2));
  const auto [S, dt] = time_grid(ttm, kHawkesStepsPerYear);
  if (int rc = launch_hawkes_slice(s.dev(0), s.dev(1), s.dev(2), nb_path, 0, use_initial_arrays ? 0 : 1, *params, S, dt, slice_index, 1.0, seed,
                                   flags, d_mom.as<double>(), st))
    return rc;
  if (int rc = s.download()) return rc;
  return sync.done();
}

// exact event-driven route (hawkes_kernels.cuh, DESIGN.md §3.13)
int b200sv_hawkesjd_mc_chain_exact(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards, const double* discfactors,
                                   const int* offsets, const double* strikes, const int8_t* types, long long nb_path, int variable_type,
                                   uint64_t seed, int flags, double* prices_out, double* stderr_out, long long max_candidates,
                                   long long n_paths_out, double* states_out, double* events_out) {
  B200SV_REQUIRE(params && ttms && forwards && discfactors && offsets && prices_out && stderr_out, "null pointer");
  return hawkes_exact_chain_host(params, M, ttms, forwards, discfactors, offsets, strikes, types, nb_path, variable_type, seed, flags, prices_out,
                                 stderr_out, max_candidates, n_paths_out, states_out, events_out);
}

int b200sv_hawkesjd_terminal_exact(const b200sv_hawkes_params* params, double ttm, long long nb_path, uint64_t seed, int flags, int slice_index,
                                   int use_initial_arrays, long long max_candidates, double* x_inout, double* lambda_p_inout,
                                   double* lambda_m_inout) {
  B200SV_REQUIRE(params && x_inout && lambda_p_inout && lambda_m_inout, "null pointer");
  B200SV_REQUIRE(nb_path >= 1 && ttm > 0.0 && slice_index >= 0, "nb_path, ttm must be positive");
  B200SV_REQUIRE(!(flags & B200SV_STATE_F32), "the Hawkes route is float64 only");
  const long long budget = hawkes_exact_budget(max_candidates);
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  HostState s(x_inout, lambda_p_inout, lambda_m_inout, nb_path, st);
  DevBuf d_mom(st), d_flag(st);
  if (int rc = s.alloc(use_initial_arrays != 0)) return rc;
  B200SV_CUDA(d_mom.alloc(sizeof(double) * 2));
  B200SV_CUDA(d_flag.alloc(sizeof(int)));
  B200SV_CUDA(cudaMemsetAsync(d_flag.p, 0, sizeof(int), st));
  if (int rc = launch_hawkes_exact_slice(s.dev(0), s.dev(1), s.dev(2), nb_path, 0, use_initial_arrays ? 0 : 1, *params, ttm, slice_index, 1.0,
                                         seed, budget, d_flag.as<int>(), nullptr, 0, d_mom.as<double>(), st))
    return rc;
  int overflow = 0;
  B200SV_CUDA(cudaMemcpyAsync(&overflow, d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200SV_CUDA(cudaStreamSynchronize(st));
  if (overflow) return fail(-6, "candidate budget exhausted: a path of the exact Hawkes route drew more than " + std::to_string(budget) +
                                    " candidates");
  if (int rc = s.download()) return rc;
  return sync.done();
}

int b200sv_hawkesjd_step_fixed(double* x, double* lambda_p, double* lambda_m, const double* W0, const double* U_P, const double* U_M,
                               const double* J_P, const double* J_M, int S, long long N, double dt, const b200sv_hawkes_params* params) {
  B200SV_REQUIRE(x && lambda_p && lambda_m && params && (S == 0 || (W0 && U_P && U_M && J_P && J_M)), "null pointer");
  B200SV_REQUIRE(S >= 0 && N >= 1 && dt > 0.0, "S, N, dt");
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  HostState s(x, lambda_p, lambda_m, N, st);
  DevBuf w(st);
  const size_t wb = sizeof(double) * (size_t)N * (size_t)std::max(S, 1), wn = (size_t)N * (size_t)std::max(S, 1);
  if (int rc = s.alloc(true)) return rc;
  B200SV_CUDA(w.alloc(5 * wb));
  double* wd = w.as<double>();
  const double* src[5] = {W0, U_P, U_M, J_P, J_M};
  if (S > 0)
    for (int k = 0; k < 5; ++k) B200SV_CUDA(cudaMemcpyAsync(wd + k * wn, src[k], wb, cudaMemcpyHostToDevice, st));
  Grid g = persistent_grid(hawkes_step_fixed_kernel, kThreads, N);
  hawkes_step_fixed_kernel<<<g.blocks, g.threads, 0, st>>>(s.dev(0), s.dev(1), s.dev(2), wd, wd + wn, wd + 2 * wn, wd + 3 * wn, wd + 4 * wn, S, N,
                                                            make_hawkes_consts(*params, dt));
  if (int rc = check_launch("hawkes_step_fixed_kernel")) return rc;
  if (int rc = s.download()) return rc;
  return sync.done();
}

int b200sv_hawkesjd_device_draws(uint64_t seed, long long path0, long long n, int slice, int S, double dt, const b200sv_hawkes_params* params,
                                 int flags, double* W0, double* U_P, double* U_M, double* J_P, double* J_M) {
  B200SV_REQUIRE(params && W0 && U_P && U_M && J_P && J_M && n >= 1 && S >= 1 && dt > 0.0, "null pointer / sizes");
  const int g = gauss_mode(flags);
  B200SV_REQUIRE(g == kGaussF32 || g == kGaussF64, "gauss flags");
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  DevBuf d(st);
  const size_t wn = (size_t)n * S;
  B200SV_CUDA(d.alloc(sizeof(double) * 5 * wn));
  double* w = d.as<double>();
  const HawkesConsts c = make_hawkes_consts(*params, dt);
  const int blocks = (int)((n + 127) / 128);
  if (g == kGaussF64)
    hawkes_device_draws_kernel<kGaussF64><<<blocks, 128, 0, st>>>(seed, (unsigned long long)path0, n, (unsigned)slice, S, c, w, w + wn, w + 2 * wn, w + 3 * wn, w + 4 * wn);
  else
    hawkes_device_draws_kernel<kGaussF32><<<blocks, 128, 0, st>>>(seed, (unsigned long long)path0, n, (unsigned)slice, S, c, w, w + wn, w + 2 * wn, w + 3 * wn, w + 4 * wn);
  if (int rc = check_launch("hawkes_device_draws_kernel")) return rc;
  double* dst[5] = {W0, U_P, U_M, J_P, J_M};
  for (int k = 0; k < 5; ++k) B200SV_CUDA(cudaMemcpyAsync(dst[k], w + k * wn, sizeof(double) * wn, cudaMemcpyDeviceToHost, st));
  return sync.done();
}

// ---- P2P mailbox (p2p.cuh) -----------------------------------------------------------------------------------------------
int b200sv_p2p_create(int world, int rank, int max_values, void** ctx_out, unsigned char* handle_out /* 64 bytes */) {
  B200SV_REQUIRE(ctx_out && handle_out, "null pointer");
  B200SV_REQUIRE(world >= 1 && world <= kMaxPeers && rank >= 0 && rank < world && max_values >= 2, "world <= 8, 0 <= rank < world, max_values >= 2");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  P2pCtx* c = new P2pCtx();
  c->world = world;
  c->rank = rank;
  c->kmax = max_values;
  c->vals_bytes = sizeof(double) * 2 * (size_t)world * max_values;
  c->published = c->consumed = 0;
  const size_t flags_bytes = sizeof(unsigned long long) * 2 * (size_t)world;
  const size_t total = c->vals_bytes + flags_bytes + 2 * sizeof(double);
  cudaError_t e = cudaMalloc((void**)&c->mail, total);
  if (e == cudaSuccess) e = cudaMemset(c->mail, 0, total);
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, c->mail);
  if (e != cudaSuccess) {
    delete c;
    return fail(-2, std::string("b200sv_p2p_create: ") + cudaGetErrorString(e));
  }
  for (int s = 0; s < kMaxPeers; ++s) c->peer[s] = nullptr;
  c->peer[rank] = c->mail;
  c->scratch = (double*)(c->mail + c->vals_bytes + flags_bytes);
  c->status = (unsigned int*)(c->scratch + 1);
  c->spin_limit = kSpinLimit;
  memcpy(handle_out, &h, 64);
  *ctx_out = c;
  return 0;
}

int b200sv_p2p_connect(void* ctx, const unsigned char* handles /* world x 64 bytes, rank order */) {
  B200SV_REQUIRE(ctx && handles, "null pointer");
  P2pCtx* c = (P2pCtx*)ctx;
  for (int s = 0; s < c->world; ++s) {
    if (s == c->rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + 64 * (size_t)s, 64);
    void* p = nullptr;
    B200SV_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    c->peer[s] = (char*)p;
  }
  return 0;
}

int b200sv_p2p_destroy(void* ctx) {
  if (!ctx) return 0;
  P2pCtx* c = (P2pCtx*)ctx;
  cudaDeviceSynchronize();
  for (int s = 0; s < c->world; ++s)
    if (s != c->rank && c->peer[s]) cudaIpcCloseMemHandle(c->peer[s]);
  cudaFree(c->mail);
  delete c;
  return 0;
}

int b200sv_p2p_set_spin_limit(void* ctx, unsigned int spins) {
  B200SV_REQUIRE(ctx && spins >= 1, "null pointer / spins");
  ((P2pCtx*)ctx)->spin_limit = spins;
  return 0;
}

// timeout bits of the exchanges since the last call (bit r: peer r did not publish within the spin limit); synchronises `stream` first
int b200sv_p2p_status(void* ctx, unsigned int* status_out, void* stream) {
  B200SV_REQUIRE(ctx && status_out, "null pointer");
  P2pCtx* c = (P2pCtx*)ctx;
  cudaStream_t st = (cudaStream_t)stream;
  B200SV_CUDA(cudaMemcpyAsync(status_out, c->status, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  B200SV_CUDA(cudaStreamSynchronize(st));
  if (*status_out) B200SV_CUDA(cudaMemsetAsync(c->status, 0, sizeof(unsigned int), st));
  return 0;
}

// test hook: account for a publish that never happens (a peer that died / never arrived) -- the next gather on this context waits for an epoch
// nobody signals and must run into the spin limit: poisoned values + status bit, never a hang
int b200sv_debug_p2p_lose_publish(void* ctx) {
  B200SV_REQUIRE(ctx, "null pointer");
  ++((P2pCtx*)ctx)->published;
  return 0;
}

int b200sv_dev_p2p_publish(void* ctx, const double* vals, int K, void* stream) {
  B200SV_REQUIRE(ctx && K >= 1, "null pointer / K");
  P2pCtx* c = (P2pCtx*)ctx;
  B200SV_REQUIRE(K <= c->kmax, "K exceeds the mailbox size");
  p2p_publish_kernel<<<1, 128, 0, (cudaStream_t)stream>>>(vals, K, make_publish(c, (cudaStream_t)stream));
  return check_launch("p2p_publish_kernel");
}

int b200sv_dev_p2p_gather(void* ctx, int K, double* out, void* stream) {
  B200SV_REQUIRE(ctx && out && K >= 1, "null pointer / K");
  P2pCtx* c = (P2pCtx*)ctx;
  B200SV_REQUIRE(K <= c->kmax, "K exceeds the mailbox size");
  p2p_gather_kernel<<<1, 128, 0, (cudaStream_t)stream>>>(make_gather(c), K, out);
  return check_launch("p2p_gather_kernel");
}

}  // extern "C"
