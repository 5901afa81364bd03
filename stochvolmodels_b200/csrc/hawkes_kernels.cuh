// hawkes_kernels.cuh -- Hawkes jump-diffusion Monte Carlo (two mutually exciting jump intensities) for sm_90a.
// Included by mc_kernels.cu (same translation unit: it reuses the payoff / reduction launchers and the Philox generator).
//
// Replaces, behind the C ABI of include/b200sv.h (/root/reference/src/stochvolmodels/pricers/hawkes_jd_pricer.py):
//   simulate_hawkesjd_terminal   :718-779   1800 steps per year (:752); per step and path: one scaled normal w0, two exponential clocks
//                                           u = -ln(U)/dt compared with the intensities (a jump fires when lambda > u, :767-768), two
//                                           shifted-exponential jump sizes; explicit Euler on (x, lambda_p, lambda_m) (:765-776)
//   hawkesjd_mc_chain_pricer     :644-715   slices chained on the terminal state, payoffs = utils/mc_payoffs.py on x
//
// Two kernels.  hawkes_step_fixed_kernel: caller-supplied (W0, U_P, U_M, J_P, J_M) [S][N] in the reference's own form, reference
// evaluation order without FMA contraction (the reference is plain numpy: IEEE operations one by one) -- the parity entry, 40 B of inputs
// per path-step from HBM.  hawkes_slice_kernel: the same update with every draw made in-kernel (no HBM traffic but the state):
//   normals      the stepper's stream (philox.cuh, counter word 3 = slice): one Philox call feeds 4 steps (float draws) or 2 (fp64 draws)
//   jump clocks  a second stream (slice | 0x80000000), one call per TWO steps; a third (slice | 0x40000000) holds the jump sizes and is only
//   and sizes    evaluated when a clock fires (~lambda dt = 0.5 % of the steps).  u = (r + 1/2) 2^-32.
// b200sv_hawkesjd_device_draws exports the in-kernel draws in the reference's form so that the fused kernel is checked path by path
// against the oracle on ITS OWN inputs.
#pragma once

namespace b200sv {

struct HawkesConsts {
  double dt, sqrt_dt, inv_dt;
  double drift_dt;            // (mu - sigma^2 / 2) dt                               (:763)
  double comp_p, comp_m;      // dt (exp(shift) / (1 - mean) - 1)                    (:760-761)
  double sigma;
  double shift_p, mean_p, shift_m, mean_m;
  double theta_p, kappa_p, beta1_p, beta2_p, theta_m, kappa_m, beta1_m, beta2_m;
};

static HawkesConsts make_hawkes_consts(const b200sv_hawkes_params& p, double dt) {
  HawkesConsts c;
  c.dt = dt;
  c.sqrt_dt = std::sqrt(dt);
  c.inv_dt = 1.0 / dt;
  c.drift_dt = (p.mu - 0.5 * p.sigma * p.sigma) * dt;
  c.comp_p = dt * (std::exp(p.shift_p) / (1.0 - p.mean_p) - 1.0);
  c.comp_m = dt * (std::exp(p.shift_m) / (1.0 - p.mean_m) - 1.0);
  c.sigma = p.sigma;
  c.shift_p = p.shift_p;
  c.mean_p = p.mean_p;
  c.shift_m = p.shift_m;
  c.mean_m = p.mean_m;
  c.theta_p = p.theta_p;
  c.kappa_p = p.kappa_p;
  c.beta1_p = p.beta1_p;
  c.beta2_p = p.beta2_p;
  c.theta_m = p.theta_m;
  c.kappa_m = p.kappa_m;
  c.beta1_m = p.beta1_m;
  c.beta2_m = p.beta2_m;
  return c;
}

// one Euler step in the reference's evaluation order (:765-776), IEEE operations without contraction
__device__ __forceinline__ void hawkes_update(double& x, double& lp, double& lm, double w0, double jump_p, double jump_m, const HawkesConsts& c) {
  const double diffusion = __dadd_rn(__dadd_rn(__dadd_rn(c.drift_dt, -__dmul_rn(c.comp_p, lp)), -__dmul_rn(c.comp_m, lm)), __dmul_rn(c.sigma, w0));
  x = __dadd_rn(__dadd_rn(__dadd_rn(x, diffusion), jump_p), jump_m);
  const double load_p = __dadd_rn(__dmul_rn(c.beta1_p, jump_p), __dmul_rn(c.beta2_p, jump_m));
  const double load_m = __dadd_rn(__dmul_rn(c.beta1_m, jump_p), __dmul_rn(c.beta2_m, jump_m));
  lp = __dadd_rn(__dadd_rn(lp, __dmul_rn(__dmul_rn(c.kappa_p, __dadd_rn(c.theta_p, -lp)), c.dt)), load_p);
  lm = __dadd_rn(__dadd_rn(lm, __dmul_rn(__dmul_rn(c.kappa_m, __dadd_rn(c.theta_m, -lm)), c.dt)), load_m);
}

__global__ void __launch_bounds__(kThreads) hawkes_step_fixed_kernel(double* __restrict__ x, double* __restrict__ lam_p, double* __restrict__ lam_m,
                                                                    const double* __restrict__ W0, const double* __restrict__ U_P,
                                                                    const double* __restrict__ U_M, const double* __restrict__ J_P,
                                                                    const double* __restrict__ J_M, int S, long long N, HawkesConsts c) {
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < N; i += stride) {
    double xi = x[i], lp = lam_p[i], lm = lam_m[i];
    for (int s = 0; s < S; ++s) {
      const size_t o = (size_t)s * N + i;
      const double jp = lp > __ldg(U_P + o) ? __ldg(J_P + o) : 0.0;       // np.where(lambda_p0 > u_p, j_p, 0.0)
      const double jm = lm > __ldg(U_M + o) ? __ldg(J_M + o) : 0.0;
      hawkes_update(xi, lp, lm, __ldg(W0 + o), jp, jm, c);
    }
    x[i] = xi;
    lam_p[i] = lp;
    lam_m[i] = lm;
  }
}

// Jump streams of one path (counter word 3 = slice | flag; the stepper's normals use the plain slice):
//   clocks  flag 0x80000000, call k = step / 2:  words (x, y) = the (+, -) clocks of step 2k, (z, w) = those of step 2k + 1
//   sizes   flag 0x40000000, call = step:        words (x, y) = the (+, -) jump sizes -- evaluated only when a clock fires
// uniform in (0, 1) of a 32-bit word: (r + 1/2) 2^-32
__device__ __forceinline__ uint4 hawkes_clock_words(uint2 key, uint32_t plo, uint32_t phi, uint32_t pair, uint32_t slice) {
  return philox4x32_10(make_uint4(plo, phi, pair, slice | 0x80000000u), key);
}
__device__ __forceinline__ uint4 hawkes_size_words(uint2 key, uint32_t plo, uint32_t phi, uint32_t step, uint32_t slice) {
  return philox4x32_10(make_uint4(plo, phi, step, slice | 0x40000000u), key);
}
__device__ __forceinline__ double hawkes_uniform(uint32_t r) { return fma((double)r, 2.3283064365386963e-10, 1.1641532182693481e-10); }
// exponential clock -ln(U)/dt and shifted-exponential sizes exactly as b200sv_hawkesjd_device_draws exports them
__device__ __forceinline__ double hawkes_clock(double u, const HawkesConsts& c) { return __ddiv_rn(-log(u), c.dt); }
__device__ __forceinline__ double hawkes_size_p(double u, const HawkesConsts& c) { return __dadd_rn(c.shift_p, __dmul_rn(c.mean_p, -log(u))); }
__device__ __forceinline__ double hawkes_size_m(double u, const HawkesConsts& c) { return __dadd_rn(c.shift_m, -__dmul_rn(-c.mean_m, -log(u))); }

struct HawkesSliceArgs {
  double *x, *lam_p, *lam_m;
  long long n;
  unsigned long long path_offset;
  int init;                    // 1: start every path from (0, lambda_p0, lambda_m0)
  double lam_p0, lam_m0;
  int nsteps;
  unsigned int slice;
  unsigned long long seed;
  double forward;
  double* partials;            // [gridDim.x][2]: (sum F e^x over non-NaN, count) for the forward re-centring
};

// Throughput stepper.  Per step the common case (no jump, ~99.5 % of the steps at the reference's parameters) is 8 contracted fp64
// operations; whether a clock CAN fire is decided on the raw 32-bit word: -ln(u) >= 1 - u, so a jump needs 1 - u < lambda dt, i.e.
// r >= floor(2^32 (1 - lambda dt (1 + 1e-9))) - 1 (one DFMA + F2I + integer compare; the margins cover the rounding of the product and of
// the floor, tests/test_gpu_hawkes_edges.py checks the filter at its edge words).  Only then are the logarithm, the exact comparison
// lambda > -ln(u)/dt of the reference (:767-768) and -- if it fires -- the size stream evaluated.  Same draws as b200sv_hawkesjd_device_draws
// exports; agreement with the strict kernel ~1e-15 (FMA contraction).
struct HawkesFast {
  double ssd;                // sigma sqrt(dt)
  double kdt_p, kdt_m;       // kappa dt
  double thr;                // dt (1 + 1e-9) 2^32
  double dt_lo;              // dt (1 - 1e-9)
};

// Does the clock with word r fire against intensity lam, i.e. is lam > -ln(u)/dt as the reference evaluates it (:767-768)?  With e = 1 - u
// (exact in fp64): -ln(u) <= e + e^2 for e <= 1/2, so e + e^2 < lam dt (1 - 1e-9) settles it without a logarithm; the band in between
// (relative width ~e, i.e. ~0.5 % of the candidates) takes the exact comparison, out of line.  tests/test_gpu_hawkes_edges.py checks the
// bound on both sides of its edge and at lam dt up to 50, where e + e^2 alone would accept wrongly beyond e ~ 0.68.
__device__ __noinline__ bool hawkes_fires_exact(double lam, double u, double dt) { return lam > __ddiv_rn(-log(u), dt); }
__device__ __forceinline__ bool hawkes_fires(double lam, uint32_t r, double dt, double dt_lo) {
  const double u = hawkes_uniform(r), e = 1.0 - u;
  if (e <= 0.5 && fma(e, e, e) < lam * dt_lo) return true;
  return hawkes_fires_exact(lam, u, dt);
}
// Can the clock with word r fire against lam at all (the filter above)?  fma(-lam, thr, 2^32) converts with saturation: lam <= 0 and
// lam thr < 1 give UINT_MAX (only the two top words pass), lam dt >= 1 gives 0, which max(., 1) - 1 keeps at 0 (every word passes).
__device__ __forceinline__ bool hawkes_candidate(double lam, uint32_t r, const HawkesFast& f) {
  const uint32_t t = __double2uint_rd(fma(-lam, f.thr, 4294967296.0));
  return r >= max(t, 1u) - 1u;
}
// The stepper's firing decision is hawkes_candidate(lam, r, f) && hawkes_fires(lam, r, dt, dt_lo), == (lam > hawkes_clock(hawkes_uniform(r))).
// It is written out at its call sites rather than wrapped: any function layer around the && changes the slice kernels' machine code.
// both clocks firing in one step (~1e-5 of the steps): out of line
__device__ __noinline__ double2 hawkes_two_sizes(uint32_t wx, uint32_t wy, double shift_p, double mean_p, double shift_m, double mean_m) {
  return make_double2(__dadd_rn(shift_p, __dmul_rn(mean_p, -log(hawkes_uniform(wx)))), __dadd_rn(shift_m, -__dmul_rn(-mean_m, -log(hawkes_uniform(wy)))));
}

#ifndef B200SV_HAWKES_MINBLOCKS
#define B200SV_HAWKES_MINBLOCKS 2
#endif
// Observer of the stepper (DESIGN.md §3.11).  step() sees every step after the primal update with the intensities the firing test read,
// the normal, the two firing decisions and the jump sizes.  The default observes nothing and compiles away, so hawkes_slice_kernel is the
// same machine code with or without this hook.
struct HawkesNoHook {
  __device__ __forceinline__ void step(double, double, double, bool, bool, double, double) {}
};

// the S steps of one path of one slice from (xi, lp, lm): the draws and the update of hawkes_slice_kernel
template <int GAUSS, class Hook>
__device__ __forceinline__ void hawkes_path_steps(double& xi, double& lp, double& lm, const HawkesSliceArgs& a, const HawkesConsts& c,
                                                  const HawkesFast& f, uint2 key, uint32_t plo, uint32_t phi, StepNormals<double, GAUSS>& rng,
                                                  Hook& hk) {
  auto one_step = [&](double z, uint32_t rp, uint32_t rm, uint32_t step) {
    const double lp0 = lp, lm0 = lm;
    const bool cand_p = hawkes_candidate(lp, rp, f), cand_m = hawkes_candidate(lm, rm, f);
    double jp = 0.0, jm = 0.0;
    bool fp_ = false, fm_ = false;
    if (cand_p || cand_m) {                                                     // ~1 % of the lane-steps: a clock may fire
      fp_ = cand_p && hawkes_fires(lp, rp, c.dt, f.dt_lo);
      fm_ = cand_m && hawkes_fires(lm, rm, c.dt, f.dt_lo);
      if (fp_ || fm_) {
        const uint4 w = hawkes_size_words(key, plo, phi, step, a.slice);
        if (fp_ && fm_) {
          const double2 jj = hawkes_two_sizes(w.x, w.y, c.shift_p, c.mean_p, c.shift_m, c.mean_m);
          jp = jj.x;
          jm = jj.y;
        } else {                                                                // one logarithm serves whichever clock fired
          const double l = -log(hawkes_uniform(fp_ ? w.x : w.y));
          if (fp_) jp = __dadd_rn(c.shift_p, __dmul_rn(c.mean_p, l));            // = hawkes_size_p
          else jm = __dadd_rn(c.shift_m, -__dmul_rn(-c.mean_m, l));              // = hawkes_size_m
        }
      }
    }
    double d = fma(-c.comp_p, lp, c.drift_dt);
    d = fma(-c.comp_m, lm, d);
    d = fma(f.ssd, z, d);
    xi += d;
    lp = fma(f.kdt_p, c.theta_p - lp, lp);
    lm = fma(f.kdt_m, c.theta_m - lm, lm);
    if (jp != 0.0 || jm != 0.0) {
      xi += jp + jm;
      lp += fma(c.beta1_p, jp, c.beta2_p * jm);
      lm += fma(c.beta1_m, jp, c.beta2_m * jm);
    }
    hk.step(lp0, lm0, z, fp_, fm_, jp, jm);
  };
  const int S = a.nsteps;
  for (int s = 0; s < S; s += 4) {                  // four steps: one (float) or two (fp64) calls of normals, two calls of clocks
    double z[4];
    if constexpr (GAUSS == kGaussF64) {
      rng.get((uint32_t)(s >> 1), z[0], z[1]);
      if (s + 2 < S) rng.get((uint32_t)(s >> 1) + 1u, z[2], z[3]);
    } else {
      rng.get2((uint32_t)(s >> 2), z[0], z[1], z[2], z[3]);
    }
    const uint4 c0 = hawkes_clock_words(key, plo, phi, (uint32_t)(s >> 1), a.slice);
    one_step(z[0], c0.x, c0.y, (uint32_t)s);
    if (s + 1 < S) one_step(z[1], c0.z, c0.w, (uint32_t)s + 1u);
    if (s + 2 < S) {
      const uint4 c1 = hawkes_clock_words(key, plo, phi, (uint32_t)(s >> 1) + 1u, a.slice);
      one_step(z[2], c1.x, c1.y, (uint32_t)s + 2u);
      if (s + 3 < S) one_step(z[3], c1.z, c1.w, (uint32_t)s + 3u);
    }
  }
}

__device__ __forceinline__ HawkesFast hawkes_fast(const HawkesConsts& c) {
  return HawkesFast{c.sigma * c.sqrt_dt, c.kappa_p * c.dt, c.kappa_m * c.dt, c.dt * (1.0 + 1e-9) * 4294967296.0, c.dt * (1.0 - 1e-9)};
}

template <int GAUSS>
__global__ void __launch_bounds__(kThreads, B200SV_HAWKES_MINBLOCKS) hawkes_slice_kernel(HawkesSliceArgs a, HawkesConsts c) {
  if constexpr (GAUSS != kGaussF32) gauss64_table_init();
  SpotMoments<2, kThreads> mom;
  const uint2 key = make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32));
  const HawkesFast f = hawkes_fast(c);
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < a.n; i += stride) {
    double xi = 0.0, lp = a.lam_p0, lm = a.lam_m0;
    if (!a.init) {
      xi = a.x[i];
      lp = a.lam_p[i];
      lm = a.lam_m[i];
    }
    const unsigned long long path = a.path_offset + (unsigned long long)i;
    const uint32_t plo = (uint32_t)path, phi = (uint32_t)(path >> 32);
    StepNormals<double, GAUSS> rng(a.seed, path, a.slice);
    HawkesNoHook none;
    hawkes_path_steps<GAUSS>(xi, lp, lm, a, c, f, key, plo, phi, rng, none);
    a.x[i] = xi;
    a.lam_p[i] = lp;
    a.lam_m[i] = lm;
    mom.add(a.forward * exp(xi));
  }
  mom.store(a.partials);
}
// ---- Monte Carlo sensitivities (DESIGN.md §3.11) -----------------------------------------------------------------------------
// Directions in HAWKES_GREEK_PARAMS order: 0 sigma, 1 shift_p, 2 mean_p, 3 shift_m, 4 mean_m, 5..9 (lambda, theta, kappa, beta1, beta2)_p,
// 10..14 the same for the minus intensity.  With the firing decisions frozen, sigma moves only x, the five own parameters of an intensity
// move only that intensity, and the shifts and means move both through the jump loads: each intensity carries 9 tangents, q = 0..3 the
// shift / mean directions, q = 4..8 its own five.
constexpr int kHawkesParams = 15;
constexpr int kHawkesLamDirs = 9;
__host__ __device__ constexpr int hawkes_dir_p(int q) { return q + 1; }
__host__ __device__ constexpr int hawkes_dir_m(int q) { return q < 4 ? q + 1 : q + 6; }

// the chain's tangent state between maturities, SoA [rows][n]: dx [15], dlambda_p [9], dlambda_m [9], accumulated score [15] (row 0 is 0)
struct HawkesTangentArgs {
  double *dx, *dlp, *dlm, *score;
};

// Pathwise tangents with frozen decisions plus the likelihood-ratio score of the decisions.  dx and the no-jump score are linear in the
// step-start intensity tangents, so the hook keeps their running sums rp / rm over the slice and forms dx and the score once at the end:
//   dx_p    += -comp_p rp_p - comp_m rm_p  (+ sqrt(dt) sum z - sigma dt S for sigma, + firings - dcomp/dshift sum lambda for the shifts,
//              + sum E - dcomp/dmean sum lambda for the means, E = (J - shift) / mean the unit exponential of a jump)
//   score_p += -dt (rp_p + rm_p) + fire_p,  fire_p = sum over firing steps of dlambda (dt + dt / expm1(lambda dt)), plus dt dlambda on steps
//              with lambda <= 0 (the clock cannot fire there: no score)
struct HawkesTangentHook {
  const HawkesConsts& c;
  double a_p, a_m;                            // 1 - kappa dt: d lambda' / d lambda between jumps
  double dlp[kHawkesLamDirs], dlm[kHawkesLamDirs];
  double rp[kHawkesLamDirs], rm[kHawkesLamDirs];
  double fire[kHawkesParams];                 // index = direction; fire[0] stays 0
  double sp, sm, np_, nm_, ep, em, zs;        // sums of the step-start intensities, firing counts, sums of E, sum of z

  __device__ __forceinline__ HawkesTangentHook(const HawkesConsts& c_, const HawkesFast& f) : c(c_), a_p(1.0 - f.kdt_p), a_m(1.0 - f.kdt_m) {}

  __device__ __forceinline__ void load(const HawkesTangentArgs& t, long long i, long long n, bool init) {
#pragma unroll
    for (int q = 0; q < kHawkesLamDirs; ++q) {
      dlp[q] = init ? (q == 4 ? 1.0 : 0.0) : t.dlp[q * n + i];          // d lambda_p(0) / d lambda_p = 1
      dlm[q] = init ? (q == 4 ? 1.0 : 0.0) : t.dlm[q * n + i];
      rp[q] = rm[q] = 0.0;
    }
#pragma unroll
    for (int p = 0; p < kHawkesParams; ++p) fire[p] = 0.0;
    sp = sm = np_ = nm_ = ep = em = zs = 0.0;
  }

  __device__ __forceinline__ void step(double lp0, double lm0, double z, bool fp, bool fm, double jp, double jm) {
    zs += z;
    sp += lp0;
    sm += lm0;
    if (fp || fm || !(lp0 > 0.0) || !(lm0 > 0.0)) {           // score terms at the step-start tangents (~1 % of the lane-steps)
      const double wp = fp ? c.dt + c.dt / expm1(lp0 * c.dt) : (lp0 > 0.0 ? 0.0 : c.dt);
      const double wm = fm ? c.dt + c.dt / expm1(lm0 * c.dt) : (lm0 > 0.0 ? 0.0 : c.dt);
#pragma unroll
      for (int q = 0; q < kHawkesLamDirs; ++q) {
        fire[hawkes_dir_p(q)] = fma(wp, dlp[q], fire[hawkes_dir_p(q)]);
        fire[hawkes_dir_m(q)] = fma(wm, dlm[q], fire[hawkes_dir_m(q)]);
      }
    }
    const double kp = c.dt * (c.theta_p - lp0), km = c.dt * (c.theta_m - lm0);
#pragma unroll
    for (int q = 0; q < kHawkesLamDirs; ++q) {
      rp[q] += dlp[q];
      rm[q] += dlm[q];
      const double bp = q == 5 ? c.kappa_p * c.dt : q == 6 ? kp : 0.0;   // theta: kappa dt, kappa: dt (theta - lambda)
      const double bm = q == 5 ? c.kappa_m * c.dt : q == 6 ? km : 0.0;
      dlp[q] = fma(a_p, dlp[q], bp);
      dlm[q] = fma(a_m, dlm[q], bm);
    }
    if (fp || fm) {                                           // the jump loads: dJ/dshift = 1, dJ/dmean = E; beta rows take J itself
      const double up = fp ? 1.0 : 0.0, um = fm ? 1.0 : 0.0;
      const double eep = fp ? (jp - c.shift_p) / c.mean_p : 0.0, eem = fm ? (jm - c.shift_m) / c.mean_m : 0.0;
      np_ += up;
      nm_ += um;
      ep += eep;
      em += eem;
      dlp[0] = fma(c.beta1_p, up, dlp[0]);
      dlp[1] = fma(c.beta1_p, eep, dlp[1]);
      dlp[2] = fma(c.beta2_p, um, dlp[2]);
      dlp[3] = fma(c.beta2_p, eem, dlp[3]);
      dlp[7] += jp;
      dlp[8] += jm;
      dlm[0] = fma(c.beta1_m, up, dlm[0]);
      dlm[1] = fma(c.beta1_m, eep, dlm[1]);
      dlm[2] = fma(c.beta2_m, um, dlm[2]);
      dlm[3] = fma(c.beta2_m, eem, dlm[3]);
      dlm[7] += jp;
      dlm[8] += jm;
    }
  }

  // end of the slice (S steps): dx and the score from their values at the slice start, into the SoA state
  __device__ __forceinline__ void finish(const HawkesTangentArgs& t, long long i, long long n, bool init, int S, double (&dx)[kHawkesParams],
                                         double (&sc)[kHawkesParams]) const {
#pragma unroll
    for (int p = 0; p < kHawkesParams; ++p) {
      dx[p] = init ? 0.0 : t.dx[p * n + i];
      sc[p] = init ? 0.0 : t.score[p * n + i];
    }
    dx[0] += fma(c.sqrt_dt, zs, -c.sigma * c.dt * (double)S);
    const double gp = c.dt * exp(c.shift_p) / (1.0 - c.mean_p), gm = c.dt * exp(c.shift_m) / (1.0 - c.mean_m);   // dcomp / dshift
    dx[1] += fma(-gp, sp, np_);
    dx[2] += fma(-gp / (1.0 - c.mean_p), sp, ep);                                                                   // dcomp / dmean
    dx[3] += fma(-gm, sm, nm_);
    dx[4] += fma(-gm / (1.0 - c.mean_m), sm, em);
#pragma unroll
    for (int q = 0; q < kHawkesLamDirs; ++q) {
      dx[hawkes_dir_p(q)] = fma(-c.comp_p, rp[q], dx[hawkes_dir_p(q)]);
      dx[hawkes_dir_m(q)] = fma(-c.comp_m, rm[q], dx[hawkes_dir_m(q)]);
      sc[hawkes_dir_p(q)] = fma(-c.dt, rp[q], sc[hawkes_dir_p(q)]);
      sc[hawkes_dir_m(q)] = fma(-c.dt, rm[q], sc[hawkes_dir_m(q)]);
    }
#pragma unroll
    for (int p = 1; p < kHawkesParams; ++p) sc[p] += fire[p];
#pragma unroll
    for (int q = 0; q < kHawkesLamDirs; ++q) {
      t.dlp[q * n + i] = dlp[q];
      t.dlm[q * n + i] = dlm[q];
    }
#pragma unroll
    for (int p = 0; p < kHawkesParams; ++p) {
      t.dx[p * n + i] = dx[p];
      t.score[p * n + i] = sc[p];
    }
  }
};

// hawkes_slice_kernel with tangents and scores: the same primal steps (bit-identical state), the same Philox streams, launched on the
// pricing kernel's grid so that the re-centring moments (first two partials) are the pricing route's.  Per-CTA partials [gridDim.x][2 + 15]:
// sum F e^x, count, sum F e^x (dx_p + score_p) over the non-NaN spots.
template <int GAUSS>
__global__ void __launch_bounds__(kThreads) hawkes_tangent_slice_kernel(HawkesSliceArgs a, HawkesConsts c, HawkesTangentArgs t) {
  constexpr int K = 2 + kHawkesParams;
  __shared__ double red[K * kThreads / 32];
  if constexpr (GAUSS != kGaussF32) gauss64_table_init();
  double acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.0;
  const uint2 key = make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32));
  const HawkesFast f = hawkes_fast(c);
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < a.n; i += stride) {
    double xi = 0.0, lp = a.lam_p0, lm = a.lam_m0;
    if (!a.init) {
      xi = a.x[i];
      lp = a.lam_p[i];
      lm = a.lam_m[i];
    }
    const unsigned long long path = a.path_offset + (unsigned long long)i;
    const uint32_t plo = (uint32_t)path, phi = (uint32_t)(path >> 32);
    StepNormals<double, GAUSS> rng(a.seed, path, a.slice);
    HawkesTangentHook h(c, f);
    h.load(t, i, a.n, a.init != 0);
    hawkes_path_steps<GAUSS>(xi, lp, lm, a, c, f, key, plo, phi, rng, h);
    a.x[i] = xi;
    a.lam_p[i] = lp;
    a.lam_m[i] = lm;
    double dx[kHawkesParams], sc[kHawkesParams];
    h.finish(t, i, a.n, a.init != 0, a.nsteps, dx, sc);
    const double spot = a.forward * exp(xi);
    if (spot == spot) {
      acc[0] += spot;
      acc[1] += 1.0;
#pragma unroll
      for (int k = 0; k < kHawkesParams; ++k) acc[2 + k] = fma(spot, dx[k] + sc[k], acc[2 + k]);
    }
  }
  block_sum<K, kThreads>(acc, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) a.partials[K * blockIdx.x + k] = acc[k];
  }
}

// the in-kernel draws of the slice kernel in the reference's form: W0 = sqrt(dt) z, U = -ln(u)/dt, J = shift +- mean (-ln(u))   [S][n] each
template <int GAUSS>
__global__ void hawkes_device_draws_kernel(unsigned long long seed, unsigned long long path0, long long n, unsigned int slice, int S, HawkesConsts c,
                                           double* __restrict__ W0, double* __restrict__ U_P, double* __restrict__ U_M,
                                           double* __restrict__ J_P, double* __restrict__ J_M) {
  if constexpr (GAUSS != kGaussF32) gauss64_table_init();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long path = path0 + (unsigned long long)i;
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  StepNormals<double, GAUSS> rng(seed, path, slice);
  double z[4];
  for (int s = 0; s < S; ++s) {
    if constexpr (GAUSS == kGaussF64) {
      if ((s & 1) == 0) rng.get((uint32_t)(s >> 1), z[0], z[1]);
    } else {
      if ((s & 3) == 0) rng.get2((uint32_t)(s >> 2), z[0], z[1], z[2], z[3]);
    }
    const uint4 ck = hawkes_clock_words(key, (uint32_t)path, (uint32_t)(path >> 32), (uint32_t)(s >> 1), slice);
    const uint4 sz = hawkes_size_words(key, (uint32_t)path, (uint32_t)(path >> 32), (uint32_t)s, slice);
    const size_t o = (size_t)s * n + i;
    W0[o] = __dmul_rn(c.sqrt_dt, GAUSS == kGaussF64 ? z[s & 1] : z[s & 3]);
    U_P[o] = hawkes_clock(hawkes_uniform((s & 1) ? ck.z : ck.x), c);
    U_M[o] = hawkes_clock(hawkes_uniform((s & 1) ? ck.w : ck.y), c);
    J_P[o] = hawkes_size_p(hawkes_uniform(sz.x), c);
    J_M[o] = hawkes_size_m(hawkes_uniform(sz.y), c);
  }
}

// jump-clock self-test kernel (tests): per (word, intensity) pair out[6i..6i+5] = u, hawkes_clock(u), hawkes_size_p(u), hawkes_size_m(u),
// the candidate flag and the stepper's firing decision, through the device functions hawkes_path_steps runs
__global__ void hawkes_clocks_kernel(const uint32_t* __restrict__ r, const double* __restrict__ lam, long long n, HawkesConsts c,
                                     double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const HawkesFast f = hawkes_fast(c);
  const uint32_t w = r[i];
  const double l = lam[i], u = hawkes_uniform(w);
  const bool cand = hawkes_candidate(l, w, f);
  out[6 * i] = u;
  out[6 * i + 1] = hawkes_clock(u, c);
  out[6 * i + 2] = hawkes_size_p(u, c);
  out[6 * i + 3] = hawkes_size_m(u, c);
  out[6 * i + 4] = cand ? 1.0 : 0.0;
  out[6 * i + 5] = cand && hawkes_fires(l, w, c.dt, f.dt_lo) ? 1.0 : 0.0;            // the decision of hawkes_path_steps' one_step
}

// one slice of the pricing kernel, or with `tan` of the tangent kernel on the same grid (moments_out then holds 2 + 15 values)
static int launch_hawkes_slice(double* x, double* lp, double* lm, long long n, long long path_offset, int init, const b200sv_hawkes_params& p,
                               int nsteps, double dt, int slice_index, double forward, uint64_t seed, int flags, double* moments_out,
                               cudaStream_t st, P2pCtx* p2p = nullptr, const HawkesTangentArgs* tan = nullptr) {
  const int g = gauss_mode(flags);
  if (g != kGaussF32 && g != kGaussF64) return fail(-1, "invalid argument: gauss flags");
  HawkesSliceArgs a;
  a.x = x;
  a.lam_p = lp;
  a.lam_m = lm;
  a.n = n;
  a.path_offset = (unsigned long long)path_offset;
  a.init = init;
  a.lam_p0 = p.lambda_p;
  a.lam_m0 = p.lambda_m;
  a.nsteps = nsteps;
  a.slice = (unsigned int)slice_index;
  a.seed = seed;
  a.forward = forward;
  const HawkesConsts c = make_hawkes_consts(p, dt);
  const Grid grid = persistent_grid(hawkes_slice_kernel<kGaussF32>, kThreads, n);
  return slice_moments(tan ? "hawkes_tangent_slice_kernel" : "hawkes_slice_kernel", tan ? 2 + kHawkesParams : 2, grid.blocks, moments_out, st, p2p,
                       [&](double* partials) {
                         a.partials = partials;
                         if (tan) {
                           if (g == kGaussF64)
                             hawkes_tangent_slice_kernel<kGaussF64><<<grid.blocks, grid.threads, 0, st>>>(a, c, *tan);
                           else
                             hawkes_tangent_slice_kernel<kGaussF32><<<grid.blocks, grid.threads, 0, st>>>(a, c, *tan);
                         } else if (g == kGaussF64) {
                           hawkes_slice_kernel<kGaussF64><<<grid.blocks, grid.threads, 0, st>>>(a, c);
                         } else {
                           hawkes_slice_kernel<kGaussF32><<<grid.blocks, grid.threads, 0, st>>>(a, c);
                         }
                       });
}

constexpr int kHawkesStepsPerYear = 5 * 360;     // hawkes_jd_pricer.py:752

static int hawkes_chain_host(const b200sv_hawkes_params* p, int M, const double* ttms, const double* forwards, const double* discfactors,
                             const int* offsets, const double* strikes, const int8_t* types, long long nb_path, int variable_type, uint64_t seed,
                             int flags, double* prices_out, double* stderr_out) {
  B200SV_REQUIRE(nb_path >= 1, "nb_path must be >= 1");
  B200SV_REQUIRE(!(flags & B200SV_STATE_F32), "the Hawkes route is float64 only");
  if (int rc = validate_chain(M, ttms, offsets, strikes, types, variable_type)) return rc;
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  DevBuf d(st);
  ChainIO io(1, M, ttms, forwards, discfactors, offsets, types, variable_type, st);
  const size_t N = (size_t)nb_path;
  B200SV_CUDA(d.alloc(sizeof(double) * 3 * N));
  if (int rc = io.upload(strikes)) return rc;
  double* x = d.as<double>();
  for (int m = 0; m < M; ++m) {
    const auto [S, dt] = maturity_grid(ttms, m, kHawkesStepsPerYear);
    if (int rc = launch_hawkes_slice(x, x + N, x + 2 * N, nb_path, 0, m == 0, *p, S, dt, m, forwards[m], seed, flags, io.moments(), st)) return rc;
    // compute_mc_vars_payoff(x0=x0, sigma0=x0, qvar0=x0, ...) (:703): the log-return array stands in for every argument
    if (int rc = io.payoff(0, m, x, x, false, nb_path, (double)nb_path, false)) return rc;
  }
  return io.copy_back(sync, prices_out, stderr_out, nullptr);
}

// Chain with Monte Carlo sensitivities (DESIGN.md §3.11): per maturity the tangent slice, the sensitivity rows from the score-aware payoff
// kernel and the price rows from the pricing route's own payoff launches on the same state, so prices and std errors are bit-identical to
// hawkes_chain_host.  The device state is [3 + 15 + 9 + 9 + 15][N] rows (x, lambda_p, lambda_m, dx, dlambda_p, dlambda_m, score); the first
// n_paths_out columns are copied out per maturity when states_out [M][3][n_out] or tangents_out [M][4][15][n_out] is given.
static int hawkes_chain_greeks_host(const b200sv_hawkes_params* p, int M, const double* ttms, const double* forwards, const double* discfactors,
                                    const int* offsets, const double* strikes, const int8_t* types, long long nb_path, int variable_type,
                                    uint64_t seed, int flags, double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out,
                                    long long n_paths_out, double* states_out, double* tangents_out) {
  constexpr int NP = kHawkesParams, L = kHawkesLamDirs, R = 3 + NP + 2 * L + NP;
  B200SV_REQUIRE(nb_path >= 1, "nb_path must be >= 1");
  B200SV_REQUIRE(n_paths_out >= 0 && n_paths_out <= nb_path, "n_paths_out must be in [0, nb_path]");
  // d J / d mean = (J - shift) / mean, the jump's unit exponential: undefined for a degenerate jump size
  B200SV_REQUIRE(p && p->mean_p != 0.0 && p->mean_m != 0.0, "the Hawkes sensitivities need mean_p != 0 and mean_m != 0");
  if (int rc = validate_chain(M, ttms, offsets, strikes, types, variable_type)) return rc;
  if (variable_type != B200SV_LOG_RETURN) return fail(-4, "variable_type not implemented: the Hawkes sensitivities cover LOG_RETURN");
  const int gauss = greeks_gauss(flags);
  if (gauss < 0) return gauss;
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  const size_t N = (size_t)nb_path, no = (states_out || tangents_out) ? (size_t)n_paths_out : 0;
  DevBuf d(st);
  GreeksChainIO<NP, true> io(M, ttms, forwards, discfactors, offsets, types, variable_type, nb_path, st);
  B200SV_CUDA(d.alloc(sizeof(double) * R * N));
  if (int rc = io.upload(strikes)) return rc;
  double* x = d.as<double>();
  const HawkesTangentArgs t{x + 3 * N, x + (3 + NP) * N, x + (3 + NP + L) * N, x + (3 + NP + 2 * L) * N};
  std::vector<double> h_paths(no * R * M);
  for (int m = 0; m < M; ++m) {
    const auto [S, dt] = maturity_grid(ttms, m, kHawkesStepsPerYear);
    if (int rc = launch_hawkes_slice(x, x + N, x + 2 * N, nb_path, 0, m == 0, *p, S, dt, m, forwards[m], seed, flags, io.moments(), st, nullptr, &t))
      return rc;
    if (int rc = io.payoff(m, x, x, t.dx, t.dx, (double)nb_path, t.score)) return rc;
    if (int rc = io.ChainIO::payoff(0, m, x, x, false, nb_path, (double)nb_path, false)) return rc;
    if (no)
      B200SV_CUDA(cudaMemcpy2DAsync(h_paths.data() + no * R * m, sizeof(double) * no, x, sizeof(double) * N, sizeof(double) * no, R,
                                    cudaMemcpyDeviceToHost, st));
  }
  if (int rc = io.copy_back(sync, prices_out, stderr_out, greeks_out, greeks_se_out)) return rc;
  for (size_t m = 0; m < (size_t)M && no; ++m) {
    const double* h = h_paths.data() + no * R * m;
    if (states_out) memcpy(states_out + 3 * no * m, h, sizeof(double) * 3 * no);
    if (!tangents_out) continue;
    double* o = tangents_out + 4 * NP * no * m;                      // [4][15][n_out]: dx, dlambda_p, dlambda_m, score
    memset(o, 0, sizeof(double) * 4 * NP * no);
    memcpy(o, h + 3 * no, sizeof(double) * NP * no);
    for (int q = 0; q < L; ++q) {
      memcpy(o + (NP + hawkes_dir_p(q)) * no, h + (3 + NP + q) * no, sizeof(double) * no);
      memcpy(o + (2 * NP + hawkes_dir_m(q)) * no, h + (3 + NP + L + q) * no, sizeof(double) * no);
    }
    memcpy(o + 3 * NP * no, h + (3 + NP + 2 * L) * no, sizeof(double) * NP * no);
  }
  return 0;
}

// ---- exact event-driven route (DESIGN.md §3.13) --------------------------------------------------------------------------------
// The continuous-time limit of the Euler step above, simulated without a grid by thinning (Ogata).  Per path and maturity interval of
// length T the state (x, lambda_p, lambda_m) is carried in as the Euler chain carries it; between events both intensities move
// deterministically, lambda(s) = theta + (lambda - theta) e^{-kappa s} (toward theta for kappa > 0, away from it for kappa < 0), a clock
// fires at rate max(lambda, 0), the compensator is c lambda (c = e^shift / (1 - mean) - 1, linear in lambda as in the Euler step) and the
// Brownian part of x over the interval is one Gaussian draw.
//   bound      at each candidate's start s, per intensity the largest value of its monotone deterministic path on [s, T]: max(lambda, theta,
//              0) for kappa >= 0 (theta is its limit), max(lambda, lambda(T), 0) for kappa < 0 (it grows away from theta, largest at T);
//              Lbar = the sum of the two; Lbar = 0: no event, advance to T
//   candidate  d = E / Lbar, E = -ln(u53); s + d >= T: advance to T; else advance by d, accept '+' if v Lbar < max(lambda_p, 0), '-' if
//              v Lbar < max(lambda_p, 0) + max(lambda_m, 0), else reject
//   segment    lambda <- theta + (lambda - theta) e^{-kappa d}, int lambda += theta d + (lambda - theta) (1 - e^{-kappa d}) / kappa (d at kappa = 0)
//   end        x += (mu - sigma^2/2) T - c_p int lambda_p - c_m int lambda_m + sigma sqrt(T) z
// Draws (counter word 3 = slice | 0xC0000000, a stream none of the Euler kernel's three -- slice, | 0x80000000, | 0x40000000 -- can reach):
//   candidate k (word 2 = k): (x, y) the 53-bit uniform u53 = (((x:y) >> 11) + 1) 2^-53 in (0, 1] of the waiting time, z the thinning
//              uniform v = (z + 1/2) 2^-32, w the jump size's unit exponential -ln((w + 1/2) 2^-32), read only when the candidate is accepted
//   normal     word 2 = 0xFFFFFFFF: z = Z0 of box_muller_f64_fast (gauss64.cuh) on that block
// oracle/hawkes_exact.py restates this path by path.
constexpr unsigned int kHawkesExactStream = 0xC0000000u;
constexpr unsigned int kHawkesExactNormalCall = 0xFFFFFFFFu;
constexpr long long kHawkesExactDefaultBudget = 1ll << 20;      // candidates per path and maturity (include/b200sv.h)
constexpr long long kHawkesExactMaxBudget = 0xFFFFFFFEll;        // the candidate index is counter word 2, below the normal's word

struct HawkesExactConsts {
  double drift;                 // mu - sigma^2 / 2
  double c_p, c_m;              // e^shift / (1 - mean) - 1 = comp / dt of make_hawkes_consts
  double sigma;
  double shift_p, mean_p, shift_m, mean_m;
  double theta_p, kappa_p, beta1_p, beta2_p, theta_m, kappa_m, beta1_m, beta2_m;
};

static HawkesExactConsts make_hawkes_exact_consts(const b200sv_hawkes_params& p) {
  return HawkesExactConsts{p.mu - 0.5 * p.sigma * p.sigma,
                           std::exp(p.shift_p) / (1.0 - p.mean_p) - 1.0,
                           std::exp(p.shift_m) / (1.0 - p.mean_m) - 1.0,
                           p.sigma, p.shift_p, p.mean_p, p.shift_m, p.mean_m,
                           p.theta_p, p.kappa_p, p.beta1_p, p.beta2_p, p.theta_m, p.kappa_m, p.beta1_m, p.beta2_m};
}

struct HawkesExactArgs {
  double *x, *lam_p, *lam_m;
  long long n;
  unsigned long long path_offset;
  int init;                     // 1: start every path from (0, lambda_p0, lambda_m0)
  double lam_p0, lam_m0;
  double T, sqrt_T;             // the interval's length
  unsigned int slice;
  unsigned long long seed;
  long long budget;             // candidates per path in this interval; a path that would draw one more stops and raises *overflow
  double forward;
  double* partials;             // [gridDim.x][2]: (sum F e^x over non-NaN, count) for the forward re-centring
  int* overflow;
  double* events;               // optional [3][n_out]: accepted '+', accepted '-', candidates of local paths [0, n_out)
  long long n_out;
};

// one deterministic segment of length d of one intensity: its value at the end and its integral over the segment
__device__ __forceinline__ void hawkes_exact_decay(double& lam, double& integral, double theta, double kappa, double d) {
  const double em = expm1(-kappa * d);                       // e^{-kappa d} - 1
  const double g = kappa != 0.0 ? -em / kappa : d;           // (1 - e^{-kappa d}) / kappa
  const double dev = lam - theta;
  integral += theta * d + dev * g;
  lam = theta + dev * (1.0 + em);
}

// the bound of one intensity's firing rate max(lambda, 0) from the candidate's start to the interval end, `rest` ahead, until the next
// event: the deterministic path is monotone, so its largest value is at one end (theta, its limit, bounds it for kappa >= 0)
__device__ __forceinline__ double hawkes_exact_rate_bound(double lam, double theta, double kappa, double rest) {
  const double far = kappa >= 0.0 ? theta : theta + (lam - theta) * exp(-kappa * rest);
  return fmax(fmax(lam, far), 0.0);
}

__device__ __forceinline__ double hawkes_u53(uint32_t hi, uint32_t lo) {
  const unsigned long long b = (((unsigned long long)hi << 32) | lo) >> 11;
  return (double)(b + 1ull) * 1.1102230246251565e-16;         // 2^-53
}

__global__ void __launch_bounds__(kThreads) hawkes_exact_slice_kernel(HawkesExactArgs a, HawkesExactConsts c) {
  gauss64_table_init();
  SpotMoments<2, kThreads> mom;
  const uint2 key = make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32));
  const uint32_t tag = a.slice | kHawkesExactStream;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < a.n; i += stride) {
    double xi = 0.0, lp = a.lam_p0, lm = a.lam_m0;
    if (!a.init) {
      xi = a.x[i];
      lp = a.lam_p[i];
      lm = a.lam_m[i];
    }
    const unsigned long long path = a.path_offset + (unsigned long long)i;
    const uint32_t plo = (uint32_t)path, phi = (uint32_t)(path >> 32);
    double s = 0.0, ip = 0.0, im = 0.0;
    long long k = 0, np_ = 0, nm_ = 0;
    for (;;) {
      const double bound = hawkes_exact_rate_bound(lp, c.theta_p, c.kappa_p, a.T - s) + hawkes_exact_rate_bound(lm, c.theta_m, c.kappa_m, a.T - s);
      double d = a.T - s;
      bool cand = false;
      uint4 w = make_uint4(0u, 0u, 0u, 0u);
      if (bound > 0.0) {
        w = philox4x32_10(make_uint4(plo, phi, (uint32_t)k, tag), key);
        const double dc = -log(hawkes_u53(w.x, w.y)) / bound;
        if (s + dc < a.T) {
          d = dc;
          cand = true;
        }
      }
      if (cand && k >= a.budget) {
        atomicOr(a.overflow, 1);
        break;
      }
      hawkes_exact_decay(lp, ip, c.theta_p, c.kappa_p, d);
      hawkes_exact_decay(lm, im, c.theta_m, c.kappa_m, d);
      if (!cand) break;
      s += d;
      ++k;
      const double v = fma((double)w.z, 2.3283064365386963e-10, 1.1641532182693481e-10) * bound;
      const double pp = fmax(lp, 0.0);
      const bool fire_p = v < pp, fire_m = !fire_p && v < pp + fmax(lm, 0.0);
      if (fire_p || fire_m) {
        const double e = -log(fma((double)w.w, 2.3283064365386963e-10, 1.1641532182693481e-10));
        if (fire_p) {
          const double jump = c.shift_p + c.mean_p * e;
          xi += jump;
          lp += c.beta1_p * jump;
          lm += c.beta1_m * jump;
          ++np_;
        } else {
          const double jump = c.shift_m + c.mean_m * e;
          xi += jump;
          lp += c.beta2_p * jump;
          lm += c.beta2_m * jump;
          ++nm_;
        }
      }
    }
    double z, z1;
    box_muller_f64_fast(philox4x32_10(make_uint4(plo, phi, kHawkesExactNormalCall, tag), key), z, z1);
    xi += ((c.drift * a.T - c.c_p * ip) - c.c_m * im) + c.sigma * a.sqrt_T * z;
    a.x[i] = xi;
    a.lam_p[i] = lp;
    a.lam_m[i] = lm;
    if (i < a.n_out) {
      a.events[i] = (double)np_;
      a.events[a.n_out + i] = (double)nm_;
      a.events[2 * a.n_out + i] = (double)k;
    }
    mom.add(a.forward * exp(xi));
  }
  mom.store(a.partials);
}

// one interval of the exact route on paths [path_offset, path_offset + n), then their re-centring moments into moments_out.  events:
// [3][n_out] device rows for the first n_out local paths (n_out = 0: none).
static int launch_hawkes_exact_slice(double* x, double* lp, double* lm, long long n, long long path_offset, int init, const b200sv_hawkes_params& p,
                                     double T, int slice_index, double forward, uint64_t seed, long long budget, int* overflow, double* events,
                                     long long n_out, double* moments_out, cudaStream_t st, P2pCtx* p2p = nullptr) {
  HawkesExactArgs a;
  a.x = x;
  a.lam_p = lp;
  a.lam_m = lm;
  a.n = n;
  a.path_offset = (unsigned long long)path_offset;
  a.init = init;
  a.lam_p0 = p.lambda_p;
  a.lam_m0 = p.lambda_m;
  a.T = T;
  a.sqrt_T = std::sqrt(T);
  a.slice = (unsigned int)slice_index;
  a.seed = seed;
  a.budget = budget;
  a.forward = forward;
  a.overflow = overflow;
  a.events = events;
  a.n_out = events ? n_out : 0;
  const HawkesExactConsts c = make_hawkes_exact_consts(p);
  const Grid grid = persistent_grid(hawkes_exact_slice_kernel, kThreads, n);
  return slice_moments("hawkes_exact_slice_kernel", 2, grid.blocks, moments_out, st, p2p, [&](double* partials) {
    a.partials = partials;
    hawkes_exact_slice_kernel<<<grid.blocks, grid.threads, 0, st>>>(a, c);
  });
}

// the candidate budget of the exact entry points: <= 0 selects the default
static long long hawkes_exact_budget(long long max_candidates) {
  return max_candidates <= 0 ? kHawkesExactDefaultBudget : std::min(max_candidates, kHawkesExactMaxBudget);
}

// Chain of the exact route: hawkes_chain_host's structure (one slice launch and one payoff per maturity, one copy back) on the intervals
// ttms[m] - ttms[m - 1].  The overflow flag is read before any result is copied out: a path that ran out of candidates fails the call
// with -6 and prices_out / stderr_out stay unwritten.  states_out [M][3][n_out] and events_out [M][3][n_out] (test hooks, may be NULL):
// the state and the event counts of paths [0, n_out) after each maturity.
static int hawkes_exact_chain_host(const b200sv_hawkes_params* p, int M, const double* ttms, const double* forwards, const double* discfactors,
                                   const int* offsets, const double* strikes, const int8_t* types, long long nb_path, int variable_type,
                                   uint64_t seed, int flags, double* prices_out, double* stderr_out, long long max_candidates,
                                   long long n_paths_out, double* states_out, double* events_out) {
  B200SV_REQUIRE(nb_path >= 1, "nb_path must be >= 1");
  B200SV_REQUIRE(n_paths_out >= 0 && n_paths_out <= nb_path, "n_paths_out must be in [0, nb_path]");
  B200SV_REQUIRE(!(flags & B200SV_STATE_F32), "the Hawkes route is float64 only");
  if (int rc = validate_chain(M, ttms, offsets, strikes, types, variable_type)) return rc;
  const long long budget = hawkes_exact_budget(max_candidates);
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  DevBuf d(st), d_flag(st), d_events(st);
  ChainIO io(1, M, ttms, forwards, discfactors, offsets, types, variable_type, st);
  const size_t N = (size_t)nb_path, no = (states_out || events_out) ? (size_t)n_paths_out : 0;
  B200SV_CUDA(d.alloc(sizeof(double) * 3 * N));
  B200SV_CUDA(d_flag.alloc(sizeof(int)));
  B200SV_CUDA(d_events.alloc(sizeof(double) * 3 * std::max(no, (size_t)1)));
  B200SV_CUDA(cudaMemsetAsync(d_flag.p, 0, sizeof(int), st));
  if (int rc = io.upload(strikes)) return rc;
  double* x = d.as<double>();
  std::vector<double> h_paths(no * 6 * M);
  for (int m = 0; m < M; ++m) {
    const double T = ttms[m] - (m > 0 ? ttms[m - 1] : 0.0);
    if (int rc = launch_hawkes_exact_slice(x, x + N, x + 2 * N, nb_path, 0, m == 0, *p, T, m, forwards[m], seed, budget, d_flag.as<int>(),
                                           no ? d_events.as<double>() : nullptr, (long long)no, io.moments(), st))
      return rc;
    if (int rc = io.payoff(0, m, x, x, false, nb_path, (double)nb_path, false)) return rc;
    if (no) {
      B200SV_CUDA(cudaMemcpy2DAsync(h_paths.data() + no * 6 * m, sizeof(double) * no, x, sizeof(double) * N, sizeof(double) * no, 3,
                                    cudaMemcpyDeviceToHost, st));
      B200SV_CUDA(cudaMemcpyAsync(h_paths.data() + no * (6 * m + 3), d_events.p, sizeof(double) * 3 * no, cudaMemcpyDeviceToHost, st));
    }
  }
  int overflow = 0;
  B200SV_CUDA(cudaMemcpyAsync(&overflow, d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200SV_CUDA(cudaStreamSynchronize(st));
  if (overflow) return fail(-6, "candidate budget exhausted: a path of the exact Hawkes route drew more than " + std::to_string(budget) +
                                    " candidates in one maturity interval");
  if (int rc = io.copy_back(sync, prices_out, stderr_out, nullptr)) return rc;
  for (size_t m = 0; m < (size_t)M && no; ++m) {
    if (states_out) memcpy(states_out + 3 * no * m, h_paths.data() + no * 6 * m, sizeof(double) * 3 * no);
    if (events_out) memcpy(events_out + 3 * no * m, h_paths.data() + no * (6 * m + 3), sizeof(double) * 3 * no);
  }
  return 0;
}

}  // namespace b200sv
