// rough_kernels.cuh -- rough-LogSV multi-factor Monte Carlo (Markovian lift of the rough kernel, n <= 8 factors) for sm_90a.
// Included by mc_kernels.cu (same translation unit: it reuses the payoff / reduction launchers and the Philox generator).
//
// Replaces, behind the C ABI of include/b200sv.h (paths under /root/reference/src/stochvolmodels/pricers):
//   log_spot_full_combined (f64 branch)            rough_logsv/split_simulation.py:340-361, 466-479
//     log_spot_full_solve2_f64                     :287-337      log-spot increment from the vol increment (c1 = c2 = 1/2)
//     drift_diffus_strand_f64                      :253-284      Strang splitting D(h/2) S(h) D(h/2)
//     drift_ode_solve2                             :76-124       classical RK4 on z_i' = -x_i (z_i - v0_i) + (k1 + k2 <w,z>)(theta - <w,z>)
//     diffus_sde_solve_f64                         :231-250      exact log-normal step of <w,z>, the same shift added to every factor
//   rough_logsv_mc_chain_pricer_fixed_randoms      logsv_pricer.py:1164-1232   (every maturity RESTARTS at t = 0 on its own grid and
//                                                  consumes the first S_m rows of Z0 / Z1)
//
// One thread = one path for the whole grid; the n factor values live in registers (template on n), the only HBM traffic is the two
// normals per step in the fixed-random mode (16 B / path-step, coalesced [S][P] rows) or nothing at all in the Philox mode, plus the
// terminal state.  ~160 fp64 instructions per step at n = 3 (8 RK4 slopes, one table exponential, one MUFU-seeded sqrt): fp64-pipe bound.
// The reference kernels are compiled fastmath=True, so its own evaluation order is not fixed; agreement with it is 1e-12.
//
// Pathwise sensitivities (DESIGN.md §3.10): rough_logsv_tangent_kernel steps the same RoughPath through a hook that records the
// intermediates its tangent needs, and carries per path dv[6][N], dls[6], dy[6] for (sigma0, theta, kappa1, kappa2, beta, orthog_vol);
// the chain reuses payoff_greeks_kernel / greeks_finalize_kernel of mc_kernels.cu.  With the default hook the pricing kernel is unchanged.
#pragma once

namespace b200sv {

constexpr int kMaxRoughFactors = 8;

struct RoughConsts {
  double nodes[kMaxRoughFactors], weight[kMaxRoughFactors], wlam[kMaxRoughFactors];   // x_i, w_i, w_i x_i
  double v0;            // sigma0 / sum(w): initial value and mean-reversion anchor of EVERY factor (logsv_pricer.py:1194)
  double theta, kappa1, kappa2;
  double volvol, rho, rho_comp, inv_volvol;     // vartheta = sqrt(beta^2 + orthog_vol^2), rho = beta / vartheta (logsv_pricer.py:1197-1198)
  double wsum, w_inv, vv, w_lam_v0;             // sum w, 1 / sum w, vartheta * sum w, sum w_i x_i v0
  double h, half_h, sqrt_h, inv_h;
};

static RoughConsts make_rough_consts(const b200sv_logsv_params& p, int n, const double* weights, const double* nodes, double h) {
  RoughConsts c{};
  double wsum = 0.0;
  for (int i = 0; i < n; ++i) wsum += weights[i];
  c.v0 = p.sigma0 / wsum;
  c.w_lam_v0 = 0.0;
  for (int i = 0; i < n; ++i) {
    c.nodes[i] = nodes[i];
    c.weight[i] = weights[i];
    c.wlam[i] = weights[i] * nodes[i];
    c.w_lam_v0 += c.wlam[i] * c.v0;
  }
  c.theta = p.theta;
  c.kappa1 = p.kappa1;
  c.kappa2 = p.kappa2;
  c.volvol = std::sqrt(p.beta * p.beta + p.volvol * p.volvol);     // p.volvol carries the ORTHOGONAL vol-of-vol on this route
  c.rho = p.beta / c.volvol;
  c.rho_comp = std::sqrt(1.0 - c.rho * c.rho);
  c.inv_volvol = 1.0 / c.volvol;
  c.wsum = wsum;
  c.w_inv = 1.0 / wsum;
  c.vv = c.volvol * wsum;
  c.h = h;
  c.half_h = 0.5 * h;
  c.sqrt_h = std::sqrt(h);
  c.inv_h = 1.0 / h;
  return c;
}

// Observer of RoughPath::step: receives the intermediates of the primal step that its tangent needs (rough_logsv_tangent_kernel).
// The default observes nothing and compiles away, so the pricing kernel is the same machine code with or without this hook.
struct RoughNoHook {
  __device__ __forceinline__ void stage(int, double) {}                          // <w, z> at RK4 stage point k (0..3 first drift, 4..7 second)
  __device__ __forceinline__ void diffusion(double, double, double, double) {}   // <w, u>, the log-normal exponent before / after clamp_log, e^ex
  __device__ __forceinline__ void reset() {}                                     // the step took the reset-to-1e-6 branch
  __device__ __forceinline__ void spot(double, double, double, double) {}        // vw, volw_h, term1, term2 of the log-spot increment
};

template <int N>
struct RoughPath {
  static constexpr bool kRedrawPair = false;     // rough_run_path keeps the second normal pair of a float-draw call in registers
  double v[N];
  double ls, y;

  __device__ __forceinline__ static double wsum_of(const RoughConsts& c, const double (&z)[N]) {
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < N; ++i) s = fma(c.weight[i], z[i], s);
    return s;
  }
  // slope of the drift ODE at z (split_simulation.py:100-103)
  template <class Hook>
  __device__ __forceinline__ static void slope(const RoughConsts& c, const double (&z)[N], double (&s)[N], Hook& hk, int k) {
    const double zw = wsum_of(c, z);
    hk.stage(k, zw);
    const double g = (c.kappa1 + c.kappa2 * zw) * (c.theta - zw);
#pragma unroll
    for (int i = 0; i < N; ++i) s[i] = fma(-c.nodes[i], z[i] - c.v0, g);
  }
  // classical RK4 over a step of size hh (drift_ode_solve2, :76-124); stages k0 .. k0 + 3 for the hook
  template <class Hook>
  __device__ __forceinline__ static void drift(const RoughConsts& c, double (&z)[N], double hh, Hook& hk, int k0) {
    double s1[N], s2[N], s3[N], s4[N], t[N];
    slope(c, z, s1, hk, k0);
#pragma unroll
    for (int i = 0; i < N; ++i) t[i] = fma(0.5 * hh, s1[i], z[i]);
    slope(c, t, s2, hk, k0 + 1);
#pragma unroll
    for (int i = 0; i < N; ++i) t[i] = fma(0.5 * hh, s2[i], z[i]);
    slope(c, t, s3, hk, k0 + 2);
#pragma unroll
    for (int i = 0; i < N; ++i) t[i] = fma(hh, s3[i], z[i]);
    slope(c, t, s4, hk, k0 + 3);
#pragma unroll
    for (int i = 0; i < N; ++i) z[i] = fma(hh / 6.0, (s1[i] + 2.0 * s2[i]) + (2.0 * s3[i] + s4[i]), z[i]);
  }
  __device__ __forceinline__ void init(const RoughConsts& c) {
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = c.v0;
    ls = 0.0;
    y = 0.0;
  }
  // one time step (log_spot_full_solve2_f64, :287-337): z0 drives the volatility, z1 the orthogonal part of the spot
  __device__ __forceinline__ void step(const RoughConsts& c, double z0, double z1) {
    RoughNoHook none;
    step(c, z0, z1, none);
  }
  template <class Hook>
  __device__ __forceinline__ void step(const RoughConsts& c, double z0, double z1, Hook& hk) {
    const double vw = wsum_of(c, v);
    double w_lam_vol = 0.0;
#pragma unroll
    for (int i = 0; i < N; ++i) w_lam_vol = fma(c.wlam[i], v[i], w_lam_vol);
    // Strang splitting (:281-283)
    double u[N];
#pragma unroll
    for (int i = 0; i < N; ++i) u[i] = v[i];
    drift(c, u, c.half_h, hk, 0);
    const double yw = wsum_of(c, u);
    const double ex_raw = fma(c.vv, z0 * c.sqrt_h, -0.5 * c.vv * c.vv * c.h);
    const double ex = clamp_log(ex_raw);
    const double e = exp_table(ex);
    hk.diffusion(yw, ex_raw, ex, e);
    const double Yh = yw * e;                                                           // diffus_sde_solve_f64 (:240-243)
    const double Q = c.w_inv * (Yh - yw);
#pragma unroll
    for (int i = 0; i < N; ++i) u[i] += Q;
    drift(c, u, c.half_h, hk, 4);
    double volw_h = wsum_of(c, u);
    if (!(volw_h > 0.0)) {          // NaN or <= 0: the reference resets every factor of that path to 1e-6 (:310-312)
#pragma unroll
      for (int i = 0; i < N; ++i) u[i] = 1e-6;
      volw_h = wsum_of(c, u);
      hk.reset();
    }
    double w_lam_vol_h = 0.0;
#pragma unroll
    for (int i = 0; i < N; ++i) w_lam_vol_h = fma(c.wlam[i], u[i], w_lam_vol_h);
    const double sq_vw = vw * vw, sq_vhw = volw_h * volw_h;
    const double term1 = c.inv_volvol *
                         (((volw_h - vw) * c.inv_h + 0.5 * w_lam_vol + 0.5 * w_lam_vol_h - c.w_lam_v0) * c.w_inv - c.kappa1 * c.theta +
                          (c.kappa1 - c.kappa2 * c.theta) * (0.5 * vw + 0.5 * volw_h) + c.kappa2 * (0.5 * sq_vw + 0.5 * sq_vhw)) *
                         c.h;
    const double term2 = 0.5 * c.h * sq_vw + 0.5 * c.h * sq_vhw;
    hk.spot(vw, volw_h, term1, term2);
    ls = ls - 0.5 * term2 + c.rho * term1 + c.rho_comp * (term2 > 0.0 ? fast_sqrt(term2) : sqrt(term2)) * z1;
    y = fma(0.5 * c.h, sq_vw + sq_vhw, y);
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = u[i];
  }
  // path i's terminal state: log_spot_out / qv_out [P], vol_out [N][P] (may be nullptr)
  __device__ __forceinline__ void store(double* __restrict__ log_spot_out, double* __restrict__ vol_out, double* __restrict__ qv_out, long long P,
                                        long long i) const {
    log_spot_out[i] = ls;
    qv_out[i] = y;
    if (vol_out) {
#pragma unroll
      for (int k = 0; k < N; ++k) vol_out[(size_t)k * P + i] = v[k];
    }
  }
};

// Z0 / Z1 != nullptr: caller-supplied unit normals, row-major [S][P] (device); else in-kernel Philox draws (stream of philox.cuh with
// slice = 0 for EVERY maturity, so that maturity m consumes the first S_m steps of one fixed stream per path, as the reference does with
// the rows of Z0 / Z1).  Path: RoughPath or RoughTangentPath, anything with step(c, z0, z1).
template <int GAUSS, class Path>
__device__ __forceinline__ void rough_run_path(Path& p, const RoughConsts& c, const double* __restrict__ Z0, const double* __restrict__ Z1, int S,
                                               long long P, long long i, unsigned long long seed, unsigned long long path_offset) {
  if (Z0) {
    for (int s = 0; s < S; ++s) p.step(c, __ldg(Z0 + (size_t)s * P + i), __ldg(Z1 + (size_t)s * P + i));
  } else {
    StepNormals<double, GAUSS> rng(seed, path_offset + (unsigned long long)i, 0u);
    if constexpr (GAUSS == kGaussF64) {
      for (int s = 0; s < S; ++s) {
        double z0, z1;
        rng.get((uint32_t)s, z0, z1);
        p.step(c, z0, z1);
      }
    } else {
      for (int cidx = 0; 2 * cidx < S; ++cidx) {
        double a0, a1, b0, b1;
        rng.get2((uint32_t)cidx, a0, a1, b0, b1);
        p.step(c, a0, a1);
        if (2 * cidx + 1 < S) {
          // a register-bound path draws the pair again instead of holding the second normals across the first step (same words)
          if constexpr (Path::kRedrawPair) rng.get2((uint32_t)cidx, a0, a1, b0, b1);
          p.step(c, b0, b1);
        }
      }
    }
  }
}

// vol_out: [N][P] factor values (may be nullptr), log_spot_out / qv_out: [P].
template <int N, int GAUSS>
__global__ void __launch_bounds__(kThreads) rough_logsv_kernel(double* __restrict__ log_spot_out, double* __restrict__ vol_out,
                                                              double* __restrict__ qv_out, const double* __restrict__ Z0,
                                                              const double* __restrict__ Z1, int S, long long P, RoughConsts c,
                                                              unsigned long long seed, unsigned long long path_offset) {
  exp_table_init();
  if constexpr (GAUSS != kGaussF32) gauss64_table_init();
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < P; i += stride) {
    RoughPath<N> p;
    p.init(c);
    rough_run_path<GAUSS>(p, c, Z0, Z1, S, P, i, seed, path_offset);
    p.store(log_spot_out, vol_out, qv_out, P, i);
  }
}

// the factor count n picks the template instantiation: f(std::integral_constant<int, n>{}) for n in 1..8
template <int N = 1, class F>
static int with_factors(int n, F&& f) {
  if constexpr (N > kMaxRoughFactors)
    return fail(-1, "invalid argument: the rough-vol kernel supports 1..8 factors");
  else
    return n == N ? f(std::integral_constant<int, N>{}) : with_factors<N + 1>(n, f);
}

// Both Gauss modes launch on the grid of the fp32-draw instantiation.
static int launch_rough(int n, double* ls, double* vol, double* qv, const double* Z0, const double* Z1, int S, long long P, const RoughConsts& c,
                        uint64_t seed, long long path_offset, int gauss, cudaStream_t st) {
  return with_factors(n, [&](auto nf) {
    constexpr int N = decltype(nf)::value;
    const Grid g = persistent_grid(rough_logsv_kernel<N, kGaussF32>, kThreads, P);
    const auto kernel = gauss == kGaussF64 ? rough_logsv_kernel<N, kGaussF64> : rough_logsv_kernel<N, kGaussF32>;
    kernel<<<g.blocks, g.threads, 0, st>>>(ls, vol, qv, Z0, Z1, S, P, c, seed, (unsigned long long)path_offset);
    return check_launch("rough_logsv_kernel");
  });
}

// --------------------------------------------------------------------------------------------------------------------
// pathwise (forward-mode) sensitivities of the rough chain, DESIGN.md §3.10
// --------------------------------------------------------------------------------------------------------------------
// Directions in LOGSV_GREEK_PARAMS order: sigma0, theta, kappa1, kappa2, beta, volvol (the ORTHOGONAL vol-of-vol on this route).
// Per direction the derivatives of the RoughConsts entries the step reads; weights and nodes are inputs, not directions.
constexpr int kRoughParams = 6;

struct RoughTangentConsts {
  double dv0[kRoughParams];        // d v0 = d sigma0 / W
  double dtheta[kRoughParams], dk1[kRoughParams], dk2[kRoughParams];
  double dvv[kRoughParams];        // d (vartheta W)
  double drho[kRoughParams], drho_comp[kRoughParams];
  double dlog_vt[kRoughParams];    // d vartheta / vartheta  (d (1/vartheta) = -dlog_vt / vartheta)
  double dwlv0[kRoughParams];      // d sum w_i x_i v0
  unsigned long long* reset_count; // device counter of the paths that took the reset-to-1e-6 branch at any step
};

static RoughTangentConsts make_rough_tangent_consts(const b200sv_logsv_params& p, const RoughConsts& c) {
  RoughTangentConsts k{};
  double wlam = 0.0;
  for (int i = 0; i < kMaxRoughFactors; ++i) wlam += c.wlam[i];      // unused factors are zero in RoughConsts
  const double vt = c.volvol;
  const double dvt[kRoughParams] = {0.0, 0.0, 0.0, 0.0, p.beta / vt, p.volvol / vt};
  const double dbeta[kRoughParams] = {0.0, 0.0, 0.0, 0.0, 1.0, 0.0};
  for (int q = 0; q < kRoughParams; ++q) {
    k.dv0[q] = q == 0 ? c.w_inv : 0.0;
    k.dtheta[q] = q == 1 ? 1.0 : 0.0;
    k.dk1[q] = q == 2 ? 1.0 : 0.0;
    k.dk2[q] = q == 3 ? 1.0 : 0.0;
    k.dvv[q] = c.wsum * dvt[q];
    k.drho[q] = (dbeta[q] - c.rho * dvt[q]) / vt;
    k.drho_comp[q] = c.rho_comp > 0.0 ? -c.rho * k.drho[q] / c.rho_comp : 0.0;
    k.dlog_vt[q] = dvt[q] / vt;
    k.dwlv0[q] = wlam * k.dv0[q];
  }
  return k;
}

// The production RoughPath steps the primal; this object is its hook, records the stage sums <w, z> and the other intermediates, and then
// advances the tangents dv[q][N], dls[q], dy[q] of every direction q with the linearised step (exact derivative of the discrete map).
template <int N>
struct RoughTangentPath {
  static constexpr bool kRedrawPair = true;      // 6 (N + 2) tangent doubles: no room for two normals across a step
  RoughPath<N> p;
  double dv[kRoughParams][N], dls[kRoughParams], dy[kRoughParams];
  double zw[8], yw, ex_raw, ex, e, vw, vhw, term1, term2;
  bool was_reset, any_reset;      // this step / any step of the path took the reset-to-1e-6 branch
  const RoughTangentConsts& k;     // the kernel's __grid_constant__ parameter
  __device__ __forceinline__ explicit RoughTangentPath(const RoughTangentConsts& k_) : k(k_) {}

  __device__ __forceinline__ void stage(int s, double z) { zw[s] = z; }
  __device__ __forceinline__ void diffusion(double yw_, double ex_raw_, double ex_, double e_) {
    yw = yw_;
    ex_raw = ex_raw_;
    ex = ex_;
    e = e_;
  }
  __device__ __forceinline__ void reset() {
    was_reset = true;
    any_reset = true;
  }
  __device__ __forceinline__ void spot(double vw_, double vhw_, double t1, double t2) {
    vw = vw_;
    vhw = vhw_;
    term1 = t1;
    term2 = t2;
  }

  __device__ __forceinline__ void init(const RoughConsts& c) {
    p.init(c);
    any_reset = false;
#pragma unroll
    for (int q = 0; q < kRoughParams; ++q) {
#pragma unroll
      for (int i = 0; i < N; ++i) dv[q][i] = k.dv0[q];
      dls[q] = 0.0;
      dy[q] = 0.0;
    }
  }
  // tangent of the drift slope at a stage point with <w, z> = zw_s: ds_i = -x_i (dz_i - dv0) + dg
  __device__ __forceinline__ void slope_t(const RoughConsts& c, int q, double zs, const double (&dz)[N], double (&ds)[N]) const {
    const double dzw = RoughPath<N>::wsum_of(c, dz);
    const double dg = fma(k.dk2[q], zs, fma(c.kappa2, dzw, k.dk1[q])) * (c.theta - zs) + fma(c.kappa2, zs, c.kappa1) * (k.dtheta[q] - dzw);
#pragma unroll
    for (int i = 0; i < N; ++i) ds[i] = fma(-c.nodes[i], dz[i] - k.dv0[q], dg);
  }
  // tangent of RoughPath::drift: the same RK4 stage combination applied to the stage tangents
  __device__ __forceinline__ void drift_t(const RoughConsts& c, int q, double (&dz)[N], double hh, int s0) const {
    double acc[N], t[N], s[N];
    slope_t(c, q, zw[s0], dz, s);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      acc[i] = s[i];
      t[i] = fma(0.5 * hh, s[i], dz[i]);
    }
    slope_t(c, q, zw[s0 + 1], t, s);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      acc[i] = fma(2.0, s[i], acc[i]);
      t[i] = fma(0.5 * hh, s[i], dz[i]);
    }
    slope_t(c, q, zw[s0 + 2], t, s);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      acc[i] = fma(2.0, s[i], acc[i]);
      t[i] = fma(hh, s[i], dz[i]);
    }
    slope_t(c, q, zw[s0 + 3], t, s);
#pragma unroll
    for (int i = 0; i < N; ++i) dz[i] = fma(hh / 6.0, acc[i] + s[i], dz[i]);
  }

  __device__ __forceinline__ void step(const RoughConsts& c, double z0, double z1) {
    was_reset = false;
    p.step(c, z0, z1, *this);
    const bool clamped = ex != ex_raw;
    const double sq = term2 > 0.0 ? sqrt(term2) : 0.0, half_inv_sq = term2 > 0.0 ? 0.5 / sq : 0.0;
    const double a_mean = 0.5 * vw + 0.5 * vhw, a_sq = 0.5 * vw * vw + 0.5 * vhw * vhw;
    const double dex_unit = fma(c.sqrt_h, z0, -c.vv * c.h);                 // d ex / d vv
#pragma unroll
    for (int q = 0; q < kRoughParams; ++q) {
      double du[N];
      double dvw = 0.0, dwlv = 0.0;
#pragma unroll
      for (int i = 0; i < N; ++i) {
        du[i] = dv[q][i];
        dvw = fma(c.weight[i], du[i], dvw);
        dwlv = fma(c.wlam[i], du[i], dwlv);
      }
      drift_t(c, q, du, c.half_h, 0);
      // exact log-normal step of <w, u>: dYh = e^ex (dyw + yw dex), the shift dQ = (dYh - dyw) / W added to every factor
      const double dyw = RoughPath<N>::wsum_of(c, du);
      const double dex = clamped ? 0.0 : k.dvv[q] * dex_unit;
      const double dQ = c.w_inv * (e * fma(yw, dex, dyw) - dyw);
#pragma unroll
      for (int i = 0; i < N; ++i) du[i] += dQ;
      drift_t(c, q, du, c.half_h, 4);
      double dvhw = 0.0, dwlvh = 0.0;
#pragma unroll
      for (int i = 0; i < N; ++i) {
        if (was_reset) du[i] = 0.0;
        dvhw = fma(c.weight[i], du[i], dvhw);
        dwlvh = fma(c.wlam[i], du[i], dwlvh);
        dv[q][i] = du[i];
      }
      // log-spot increment: term1 = h / vartheta * A, term2 = h / 2 (vw^2 + volw_h^2)
      const double dsum = fma(vw, dvw, vhw * dvhw);
      const double dterm2 = c.h * dsum;
      const double dA = (((dvhw - dvw) * c.inv_h + 0.5 * dwlv + 0.5 * dwlvh) - k.dwlv0[q]) * c.w_inv -
                        fma(k.dk1[q], c.theta, c.kappa1 * k.dtheta[q]) +
                        (k.dk1[q] - fma(k.dk2[q], c.theta, c.kappa2 * k.dtheta[q])) * a_mean +
                        (c.kappa1 - c.kappa2 * c.theta) * (0.5 * dvw + 0.5 * dvhw) + fma(k.dk2[q], a_sq, c.kappa2 * dsum);
      const double dterm1 = fma(-k.dlog_vt[q], term1, c.h * c.inv_volvol * dA);
      const double dsq = fma(k.drho_comp[q], sq, c.rho_comp * dterm2 * half_inv_sq);
      dls[q] += fma(dsq, z1, fma(-0.5, dterm2, fma(k.drho[q], term1, c.rho * dterm1)));
      dy[q] += dterm2;
    }
  }
};

// rough_logsv_kernel with tangents: same persistent grid-stride loop and normals (rough_run_path), same restart at t = 0.  Writes the state
// like rough_logsv_kernel, dls_out / dqv_out [6][P], dvol_out [6][N][P] (may be nullptr), and per-CTA partials [gridDim.x][2 + 6]:
// sum F e^ls, count, sum F e^ls dls_q over the non-NaN spots (the moments payoff_greeks_kernel re-centres with).  *k.reset_count += the
// number of paths that took the reset branch at ANY step of the grid (their mass across the switch is what the pathwise rows omit, DESIGN.md
// §3.10): one atomic per such path after its last step, so that no counter is held in registers across the path loop.
template <int N, int GAUSS>
__global__ void __launch_bounds__(kThreads) rough_logsv_tangent_kernel(double* __restrict__ log_spot_out, double* __restrict__ vol_out,
                                                                      double* __restrict__ qv_out, double* __restrict__ dls_out,
                                                                      double* __restrict__ dvol_out, double* __restrict__ dqv_out,
                                                                      const double* __restrict__ Z0, const double* __restrict__ Z1, int S, long long P,
                                                                      RoughConsts c, const __grid_constant__ RoughTangentConsts k,
                                                                      unsigned long long seed, double forward, double* __restrict__ partials) {
  exp_table_init();
  if constexpr (GAUSS != kGaussF32) gauss64_table_init();
  SpotMoments<2 + kRoughParams, kThreads> mom;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < P; i += stride) {
    RoughTangentPath<N> t(k);
    t.init(c);
    rough_run_path<GAUSS>(t, c, Z0, Z1, S, P, i, seed, 0ull);
    t.p.store(log_spot_out, vol_out, qv_out, P, i);
    const double spot = forward * exp(t.p.ls);
#pragma unroll
    for (int q = 0; q < kRoughParams; ++q) {
      dls_out[(size_t)q * P + i] = t.dls[q];
      dqv_out[(size_t)q * P + i] = t.dy[q];
      if (dvol_out) {
#pragma unroll
        for (int f = 0; f < N; ++f) dvol_out[((size_t)q * N + f) * P + i] = t.dv[q][f];
      }
      mom.add_term(spot, q, t.dls[q]);
    }
    mom.add(spot);
    if (t.any_reset) atomicAdd(k.reset_count, 1ull);
  }
  mom.store(partials);
}

// one maturity of the rough chain with tangents, then moments_out[2 + 6] = (sum F e^ls, count, sum F e^ls dls_q).  Both Gauss modes launch on
// the grid of the fp32-draw instantiation: the block count fixes the order of the moments' reduction.
static int launch_rough_tangent(int n, double* ls, double* vol, double* qv, double* dls, double* dvol, double* dqv, const double* Z0,
                                const double* Z1, int S, long long P, const RoughConsts& c, const RoughTangentConsts& k, uint64_t seed, int gauss,
                                double forward, double* moments_out, cudaStream_t st) {
  return with_factors(n, [&](auto nf) {
    constexpr int N = decltype(nf)::value;
    const int blocks = persistent_grid(rough_logsv_tangent_kernel<N, kGaussF32>, kThreads, P).blocks;
    const auto kernel = gauss == kGaussF64 ? rough_logsv_tangent_kernel<N, kGaussF64> : rough_logsv_tangent_kernel<N, kGaussF32>;
    return slice_moments("rough_logsv_tangent_kernel", 2 + kRoughParams, blocks, moments_out, st, nullptr, [&](double* partials) {
      kernel<<<blocks, kThreads, 0, st>>>(ls, vol, qv, dls, dvol, dqv, Z0, Z1, S, P, c, k, seed, forward, partials);
    });
  });
}

// --------------------------------------------------------------------------------------------------------------------
// Monte Carlo theta of the rough chain, DESIGN.md §3.12
// --------------------------------------------------------------------------------------------------------------------
// Every maturity restarts at t = 0 on its own grid h = ttm / S, so d/d ttm = (1/S) d/d h over the whole path, from a zero tangent.  The
// production RoughPath steps the primal; this object is its hook (the diffusion exponent, the reset branch, vw / volw_h / term1 / term2)
// and then advances dv[N], dls, dy in h.  The two RK4 half-steps (hh = h/2) are differentiated with their explicit hh-dependence: the
// stage slopes are replayed through RoughPath::slope from the step's start value, and their tangents chained as the parameter rows chain
// them.  The exponent contributes vv z0 / (2 sqrt h) - vv^2 / 2 (0 where clamp_log clamps), term1 is differentiated in its exact-arithmetic
// form (1/vartheta) ((volw_h - vw) / W + h rest), term2 and y are proportional to h, and the reset branch has zero factor tangents.
struct RoughThetaConsts {
  double dex_a, dex_b;       // d ex_raw / d h = dex_a z0 + dex_b:  vv / (2 sqrt h), -vv^2 / 2
  double qshift;             // S / ttm: tq = dy - qshift y, the Q_VAR payoff's dU = tq / ttm
};

template <int N>
struct RoughThetaPath {
  static constexpr bool kRedrawPair = true;
  RoughPath<N> p;
  double dv[N], dls, dy;
  double ex_raw, ex, e, vw, vhw, term1, term2;
  bool was_reset;
  __device__ __forceinline__ void stage(int, double) {}
  __device__ __forceinline__ void diffusion(double, double ex_raw_, double ex_, double e_) {
    ex_raw = ex_raw_;
    ex = ex_;
    e = e_;
  }
  __device__ __forceinline__ void reset() { was_reset = true; }
  __device__ __forceinline__ void spot(double vw_, double vhw_, double t1, double t2) {
    vw = vw_;
    vhw = vhw_;
    term1 = t1;
    term2 = t2;
  }
  __device__ __forceinline__ void init(const RoughConsts& c) {
    p.init(c);
#pragma unroll
    for (int i = 0; i < N; ++i) dv[i] = 0.0;
    dls = 0.0;
    dy = 0.0;
  }
  // tangent of the drift slope at z with the parameters held: ds_i = -x_i dz_i + dg
  __device__ __forceinline__ static void slope_h(const RoughConsts& c, const double (&z)[N], const double (&dz)[N], double (&ds)[N]) {
    const double zw = RoughPath<N>::wsum_of(c, z), dzw = RoughPath<N>::wsum_of(c, dz);
    const double dg = dzw * (c.kappa2 * (c.theta - zw) - fma(c.kappa2, zw, c.kappa1));
#pragma unroll
    for (int i = 0; i < N; ++i) ds[i] = fma(-c.nodes[i], dz[i], dg);
  }
  // RoughPath::drift over hh = h/2 and its h-tangent (d hh / d h = 1/2): z, dz in, both advanced
  __device__ __forceinline__ static void drift_h(const RoughConsts& c, double (&z)[N], double (&dz)[N], double hh) {
    RoughNoHook none;
    double s[N], ds[N], acc[N], dacc[N], t[N], dt[N];
    RoughPath<N>::slope(c, z, s, none, 0);
    slope_h(c, z, dz, ds);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      acc[i] = s[i];
      dacc[i] = ds[i];
      t[i] = fma(0.5 * hh, s[i], z[i]);
      dt[i] = fma(0.5 * hh, ds[i], fma(0.25, s[i], dz[i]));
    }
    RoughPath<N>::slope(c, t, s, none, 0);
    slope_h(c, t, dt, ds);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      acc[i] = fma(2.0, s[i], acc[i]);
      dacc[i] = fma(2.0, ds[i], dacc[i]);
      t[i] = fma(0.5 * hh, s[i], z[i]);
      dt[i] = fma(0.5 * hh, ds[i], fma(0.25, s[i], dz[i]));
    }
    RoughPath<N>::slope(c, t, s, none, 0);
    slope_h(c, t, dt, ds);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      acc[i] = fma(2.0, s[i], acc[i]);
      dacc[i] = fma(2.0, ds[i], dacc[i]);
      t[i] = fma(hh, s[i], z[i]);
      dt[i] = fma(hh, ds[i], fma(0.5, s[i], dz[i]));
    }
    RoughPath<N>::slope(c, t, s, none, 0);
    slope_h(c, t, dt, ds);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      acc[i] += s[i];
      dacc[i] += ds[i];
      z[i] = fma(hh / 6.0, acc[i], z[i]);
      dz[i] = fma(hh / 6.0, dacc[i], fma(1.0 / 12.0, acc[i], dz[i]));
    }
  }
  __device__ __forceinline__ void step(const RoughConsts& c, const RoughThetaConsts& k, double z0, double z1) {
    double z[N], dz[N];
    double dvw = 0.0, dwlv = 0.0, wlv = 0.0;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      z[i] = p.v[i];
      dz[i] = dv[i];
      dvw = fma(c.weight[i], dz[i], dvw);
      dwlv = fma(c.wlam[i], dz[i], dwlv);
      wlv = fma(c.wlam[i], z[i], wlv);
    }
    was_reset = false;
    p.step(c, z0, z1, *this);
    drift_h(c, z, dz, c.half_h);
    const double yw = RoughPath<N>::wsum_of(c, z), dyw = RoughPath<N>::wsum_of(c, dz);
    const double dex = ex != ex_raw ? 0.0 : fma(k.dex_a, z0, k.dex_b);
    const double Q = c.w_inv * (yw * e - yw), dQ = c.w_inv * (e * fma(yw, dex, dyw) - dyw);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      z[i] += Q;
      dz[i] += dQ;
    }
    drift_h(c, z, dz, c.half_h);
    double dvhw = 0.0, dwlvh = 0.0, wlvh = 0.0;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      if (was_reset) {
        z[i] = 1e-6;
        dz[i] = 0.0;
      }
      dvhw = fma(c.weight[i], dz[i], dvhw);
      dwlvh = fma(c.wlam[i], dz[i], dwlvh);
      wlvh = fma(c.wlam[i], z[i], wlvh);
      dv[i] = dz[i];
    }
    const double a_mean = 0.5 * vw + 0.5 * vhw, a_sq = 0.5 * vw * vw + 0.5 * vhw * vhw, dsum = fma(vw, dvw, vhw * dvhw);
    const double rest = (0.5 * wlv + 0.5 * wlvh - c.w_lam_v0) * c.w_inv - c.kappa1 * c.theta + (c.kappa1 - c.kappa2 * c.theta) * a_mean +
                        c.kappa2 * a_sq;
    const double drest = (0.5 * dwlv + 0.5 * dwlvh) * c.w_inv + (c.kappa1 - c.kappa2 * c.theta) * (0.5 * dvw + 0.5 * dvhw) + c.kappa2 * dsum;
    const double dterm1 = c.inv_volvol * ((dvhw - dvw) * c.w_inv + fma(c.h, drest, rest));
    const double dterm2 = fma(c.h, dsum, a_sq);
    const double dsq = term2 > 0.0 ? 0.5 * dterm2 / sqrt(term2) : 0.0;
    dls += fma(c.rho_comp * dsq, z1, fma(-0.5, dterm2, c.rho * dterm1));
    dy += dterm2;
  }
};

// the theta pass of one maturity: the pricing route's grid-stride loop and normals (rough_run_path) with RoughThetaPath; writes dls_out [P]
// = d ls / d h and dq_out [P] = d y / d h - qshift y, and per-CTA partials [gridDim.x][3]: sum F e^ls, count, sum F e^ls dls
template <int N>
struct RoughThetaRunner {
  static constexpr bool kRedrawPair = RoughThetaPath<N>::kRedrawPair;
  RoughThetaPath<N> t;
  const RoughThetaConsts& k;
  __device__ __forceinline__ explicit RoughThetaRunner(const RoughThetaConsts& k_) : k(k_) {}
  __device__ __forceinline__ void step(const RoughConsts& c, double z0, double z1) { t.step(c, k, z0, z1); }
};

template <int N, int GAUSS>
__global__ void __launch_bounds__(kThreads) rough_logsv_theta_kernel(double* __restrict__ dls_out, double* __restrict__ dq_out,
                                                                    const double* __restrict__ Z0, const double* __restrict__ Z1, int S, long long P,
                                                                    RoughConsts c, RoughThetaConsts k, unsigned long long seed, double forward,
                                                                    double* __restrict__ partials) {
  exp_table_init();
  if constexpr (GAUSS != kGaussF32) gauss64_table_init();
  SpotMoments<3, kThreads> mom;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < P; i += stride) {
    RoughThetaRunner<N> r(k);
    r.t.init(c);
    rough_run_path<GAUSS>(r, c, Z0, Z1, S, P, i, seed, 0ull);
    const double spot = forward * exp(r.t.p.ls);
    dls_out[i] = r.t.dls;
    dq_out[i] = fma(-k.qshift, r.t.p.y, r.t.dy);
    mom.add_term(spot, 0, r.t.dls);
    mom.add(spot);
  }
  mom.store(partials);
}

static int launch_rough_theta(int n, double* dls, double* dq, const double* Z0, const double* Z1, int S, long long P, const RoughConsts& c,
                              double ttm, uint64_t seed, int gauss, double forward, double* moments_out, cudaStream_t st) {
  RoughThetaConsts k;
  k.dex_a = 0.5 * c.vv / c.sqrt_h;
  k.dex_b = -0.5 * c.vv * c.vv;
  k.qshift = (double)S / ttm;
  return with_factors(n, [&](auto nf) {
    constexpr int N = decltype(nf)::value;
    const int blocks = persistent_grid(rough_logsv_theta_kernel<N, kGaussF32>, kThreads, P).blocks;
    const auto kernel = gauss == kGaussF64 ? rough_logsv_theta_kernel<N, kGaussF64> : rough_logsv_theta_kernel<N, kGaussF32>;
    return slice_moments("rough_logsv_theta_kernel", 3, blocks, moments_out, st, nullptr, [&](double* partials) {
      kernel<<<blocks, kThreads, 0, st>>>(dls, dq, Z0, Z1, S, P, c, k, seed, forward, partials);
    });
  });
}

// The argument checks both rough chain drivers make after their own factor-count check, and the caller's normals: the Gauss mode, the longest
// grid Smax, and Z0 / Z1 [Smax][P] on the device (left null with in-kernel Philox draws).
struct RoughChainArgs {
  int gauss = 0, Smax = 0;
  DevBuf z0, z1;
  explicit RoughChainArgs(cudaStream_t st) : z0(st), z1(st) {}

  int check(long long nb_path, const double* Z0, const double* Z1, long long z_rows, int M, const double* ttms, const int* offsets,
            const double* strikes, const int8_t* types, int variable_type, int flags, const int* nsteps, const double* hs) {
    B200SV_REQUIRE(nb_path >= 1, "nb_path must be >= 1");
    B200SV_REQUIRE((Z0 == nullptr) == (Z1 == nullptr), "Z0 and Z1 must be supplied together");
    if (int rc = validate_chain(M, ttms, offsets, strikes, types, variable_type)) return rc;
    gauss = gauss_mode(flags);
    B200SV_REQUIRE(gauss == kGaussF32 || gauss == kGaussF64, "gauss flags");
    B200SV_REQUIRE(!(flags & B200SV_STATE_F32), "the rough-vol route is float64 only");
    for (int m = 0; m < M; ++m) {
      B200SV_REQUIRE(nsteps[m] >= 1 && hs[m] > 0.0, "nsteps / h must be positive");
      Smax = std::max(Smax, nsteps[m]);
    }
    B200SV_REQUIRE(!Z0 || z_rows >= Smax, "Z0 / Z1 have fewer rows than the longest grid");
    return 0;
  }
  int upload(const double* Z0, const double* Z1, long long nb_path) {
    if (!Z0) return 0;
    B200SV_CUDA(z0.upload(Z0, (size_t)Smax * nb_path));
    B200SV_CUDA(z1.upload(Z1, (size_t)Smax * nb_path));
    return 0;
  }
};

// host-level chain driver: B parameter sets x M maturities on ONE upload of the normals (or none at all with Philox draws)
static int rough_chain_host(const b200sv_logsv_params* params, int B, int n, const double* weights /*[B][n]*/, const double* nodes /*[B][n]*/, int M,
                            const double* ttms, const double* forwards, const double* discfactors, const int* offsets, const double* strikes,
                            const int8_t* types, long long nb_path, const int* nsteps /*[M]*/, const double* hs /*[M]*/, const double* Z0,
                            const double* Z1, long long z_rows, int variable_type, uint64_t seed, int flags, double* prices_out,
                            double* stderr_out, double* ivols_out, double* states_out /* B == 1: [M][(n+2)][P] log_spot, vol[n], qv */) {
  B200SV_REQUIRE(B >= 1 && n >= 1 && n <= kMaxRoughFactors, "B >= 1 and 1 <= n_factors <= 8");
  B200SV_REQUIRE(!states_out || B == 1, "terminal states are returned for a single parameter set");
  cudaStream_t st = current_stream();
  RoughChainArgs a(st);
  if (int rc = a.check(nb_path, Z0, Z1, z_rows, M, ttms, offsets, strikes, types, variable_type, flags, nsteps, hs)) return rc;
  ensure_pool_threshold();
  StreamSync sync(st);
  const size_t P = (size_t)nb_path;
  DevBuf d_state(st);
  ChainIO io(B, M, ttms, forwards, discfactors, offsets, types, variable_type, st);
  B200SV_CUDA(d_state.alloc(sizeof(double) * (size_t)(n + 2) * P));
  if (int rc = a.upload(Z0, Z1, nb_path)) return rc;
  if (int rc = io.upload(strikes)) return rc;
  double *d_ls = d_state.as<double>(), *d_vol = d_ls + P, *d_qv = d_ls + (size_t)(n + 1) * P;
  for (int b = 0; b < B; ++b) {
    for (int m = 0; m < M; ++m) {
      const RoughConsts c = make_rough_consts(params[b], n, weights + (size_t)b * n, nodes + (size_t)b * n, hs[m]);
      if (int rc = launch_rough(n, d_ls, d_vol, d_qv, a.z0.as<double>(), a.z1.as<double>(), nsteps[m], nb_path, c, seed, 0, a.gauss, st)) return rc;
      if (states_out)
        B200SV_CUDA(cudaMemcpyAsync(states_out + (size_t)m * (n + 2) * P, d_ls, sizeof(double) * (size_t)(n + 2) * P, cudaMemcpyDeviceToHost, st));
      // the reference hands (1, nb_path)-shaped arrays to compute_mc_vars_payoff, whose "/ sqrt(x0.shape[0])" is then "/ 1":
      // this route's std errors are discfactor * nanstd(payoff) (total_paths = 1); the moments come from the log-spots here
      if (int rc = io.payoff(b, m, d_ls, d_qv, false, nb_path, 1.0, ivols_out != nullptr, true)) return rc;
    }
  }
  return io.copy_back(sync, prices_out, stderr_out, ivols_out);
}

// chain driver with pathwise sensitivities, one parameter set: per maturity tangent kernel -> moments -> payoff_greeks_kernel<6> ->
// greeks_finalize_kernel.  Prices / "std errors" keep the route's convention (discfactor * nanstd(payoff)); greeks_se is df * std / sqrt(P).
// greeks_out / greeks_se_out [1 + 6][Jtot] (row 0 = forward delta); states_out [M][n + 2][P], tangents_out [M][6][n + 2][P], resets_out [M]
// (paths that took the reset branch at any step of maturity m's grid) may be NULL.
static int rough_chain_greeks_host(const b200sv_logsv_params& p, int n, const double* weights, const double* nodes, int M, const double* ttms,
                                   const double* forwards, const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                   long long nb_path, const int* nsteps, const double* hs, const double* Z0, const double* Z1, long long z_rows,
                                   int variable_type, uint64_t seed, int flags, double* prices_out, double* stderr_out, double* greeks_out,
                                   double* greeks_se_out, double* states_out, double* tangents_out, double* resets_out, double* theta_out = nullptr,
                                   double* theta_se_out = nullptr, long long n_paths_out = 0, double* dtheta_out = nullptr) {
  constexpr int NP = kRoughParams;
  const bool with_theta = theta_out != nullptr;
  B200SV_REQUIRE(n_paths_out >= 0 && n_paths_out <= nb_path, "n_paths_out must be in [0, nb_path]");
  B200SV_REQUIRE(n >= 1 && n <= kMaxRoughFactors, "1 <= n_factors <= 8");
  cudaStream_t st = current_stream();
  RoughChainArgs a(st);
  if (int rc = a.check(nb_path, Z0, Z1, z_rows, M, ttms, offsets, strikes, types, variable_type, flags, nsteps, hs)) return rc;
  ensure_pool_threshold();
  StreamSync sync(st);
  const size_t P = (size_t)nb_path;
  const size_t nt = dtheta_out ? (size_t)n_paths_out : 0;
  DevBuf d_state(st), d_tan(st), d_dvol(st), d_resets(st), d_theta(st);
  GreeksChainIO<NP> io(M, ttms, forwards, discfactors, offsets, types, variable_type, nb_path, st, false, with_theta);
  if (with_theta) B200SV_CUDA(d_theta.alloc(sizeof(double) * 2 * P));     // theta pass: dls, dy - S y / ttm
  B200SV_CUDA(d_state.alloc(sizeof(double) * (size_t)(n + 2) * P));
  B200SV_CUDA(d_tan.alloc(sizeof(double) * 2 * NP * P));
  if (tangents_out) B200SV_CUDA(d_dvol.alloc(sizeof(double) * (size_t)NP * n * P));
  B200SV_CUDA(d_resets.alloc(sizeof(unsigned long long) * M));
  B200SV_CUDA(cudaMemsetAsync(d_resets.p, 0, sizeof(unsigned long long) * M, st));
  if (int rc = a.upload(Z0, Z1, nb_path)) return rc;
  if (int rc = io.upload(strikes)) return rc;
  double *d_ls = d_state.as<double>(), *d_vol = d_ls + P, *d_qv = d_ls + (size_t)(n + 1) * P;
  double *d_dls = d_tan.as<double>(), *d_dqv = d_dls + NP * P, *d_dv = d_dvol.as<double>();      // d_dv: null without tangents_out
  std::vector<double> h_q(nt * M);
  for (int m = 0; m < M; ++m) {
    const RoughConsts c = make_rough_consts(p, n, weights, nodes, hs[m]);
    RoughTangentConsts k = make_rough_tangent_consts(p, c);
    k.reset_count = d_resets.as<unsigned long long>() + m;
    if (int rc = launch_rough_tangent(n, d_ls, d_vol, d_qv, d_dls, d_dv, d_dqv, a.z0.as<double>(), a.z1.as<double>(), nsteps[m], nb_path, c, k, seed,
                                      a.gauss, forwards[m], io.moments(), st))
      return rc;
    if (states_out)
      B200SV_CUDA(cudaMemcpyAsync(states_out + (size_t)m * (n + 2) * P, d_ls, sizeof(double) * (size_t)(n + 2) * P, cudaMemcpyDeviceToHost, st));
    if (tangents_out) {
      for (int q = 0; q < NP; ++q) {
        double* o = tangents_out + ((size_t)m * NP + q) * (n + 2) * P;
        B200SV_CUDA(cudaMemcpyAsync(o, d_dls + q * P, sizeof(double) * P, cudaMemcpyDeviceToHost, st));
        B200SV_CUDA(cudaMemcpyAsync(o + P, d_dv + (size_t)q * n * P, sizeof(double) * n * P, cudaMemcpyDeviceToHost, st));
        B200SV_CUDA(cudaMemcpyAsync(o + (size_t)(n + 1) * P, d_dqv + q * P, sizeof(double) * P, cudaMemcpyDeviceToHost, st));
      }
    }
    // the price row keeps the route's un-normalised std (total_paths = 1), the sensitivity rows are standard errors
    if (int rc = io.payoff(m, d_ls, d_qv, d_dls, d_dqv, 1.0)) return rc;
    if (!with_theta) continue;
    // the theta pass replays the maturity's path on the same normals; its rows re-centre with the tangent pass's (sum F e^ls, count)
    double *d_th = d_theta.as<double>(), *d_thq = d_th + P;
    if (int rc = launch_rough_theta(n, d_th, d_thq, a.z0.as<double>(), a.z1.as<double>(), nsteps[m], nb_path, c, ttms[m], seed, a.gauss, forwards[m],
                                    io.theta_moments(), st))
      return rc;
    B200SV_CUDA(cudaMemcpyAsync(io.theta_moments(), io.moments(), sizeof(double) * 2, cudaMemcpyDeviceToDevice, st));
    if (int rc = io.payoff_theta(m, d_ls, d_qv, d_th, d_thq, nsteps[m])) return rc;
    if (nt) {
      B200SV_CUDA(cudaMemcpy2DAsync(dtheta_out + 2 * nt * m, sizeof(double) * nt, d_th, sizeof(double) * P, sizeof(double) * nt, 2,
                                    cudaMemcpyDeviceToHost, st));
      B200SV_CUDA(cudaMemcpyAsync(h_q.data() + nt * m, d_qv, sizeof(double) * nt, cudaMemcpyDeviceToHost, st));
    }
  }
  std::vector<unsigned long long> h_resets(M);
  B200SV_CUDA(d_resets.download(h_resets.data(), M));
  if (int rc = io.copy_back(sync, prices_out, stderr_out, greeks_out, greeks_se_out, nullptr, nullptr, theta_out, theta_se_out)) return rc;
  for (int m = 0; m < M && resets_out; ++m) resets_out[m] = (double)h_resets[m];
  // the hook reports d y / d h: undo the payoff's shift with the maturity's y
  for (int m = 0; m < M; ++m)
    for (size_t i = 0; i < nt; ++i) dtheta_out[(2 * m + 1) * nt + i] += (double)nsteps[m] / ttms[m] * h_q[nt * m + i];
  return 0;
}

}  // namespace b200sv
