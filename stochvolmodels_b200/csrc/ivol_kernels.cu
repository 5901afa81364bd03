// ivol_kernels.cu -- batched Black-76 implied-volatility inversion (SURVEY.md §8f "next" #1).
//
// In the reference this step is third-party (vanilla_option_pricers.infer_bsm_ivols_from_model_chain_prices, called from
// data/option_chain.py:327-346 right after every price_chain / model_mc_price_chain in compute_chain_prices_with_vols,
// model_pricer.py:109-120, and compute_mc_chain_implied_vols, :216-241).  That package is not in the reference tree, so bit-level
// parity with it is unpinned (DESIGN.md §2); what the reference pins -- the quickstart vols 0.999577 / 0.995757 and flat-vol
// round trips -- holds for any correct inversion; the reference's own assertions about the step (flat-vol recovery 1e-10, chain round trip
// 2e-10, single-option round trip 2e-12, slice / vanilla self-consistency 1e-12) are ported in tests/test_gpu_ivol_pins.py.  One thread per
// quote: safeguarded Newton in total-vol space (black.cuh), fp64 normcdf; the checker oracle/bsm.py is an independent 80-step bisection
// plus a numpy restatement of the Newton iteration.
#include <cmath>
#include <vector>

#include "../../include/b200sv.h"
#include "common.cuh"
#include "black.cuh"

namespace b200sv {

struct QuoteSpec {
  double forward, strike, ttm, discfactor, price;
  int type;
};

__global__ void black_ivol_kernel(const QuoteSpec* __restrict__ q, int n, double* __restrict__ ivols) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const QuoteSpec s = q[i];
  ivols[i] = black_implied_vol(s.forward, s.strike, s.ttm, s.discfactor, s.price, s.type);
}

// debug twin: the same inversion, plus the number of iterations it took (tests read the worst case; the product never counts)
__global__ void black_ivol_count_kernel(const QuoteSpec* __restrict__ q, int n, double* __restrict__ ivols, int* __restrict__ iterations) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const QuoteSpec s = q[i];
  int it;
  ivols[i] = black_implied_vol(s.forward, s.strike, s.ttm, s.discfactor, s.price, s.type, &it);
  iterations[i] = it;
}

// Implied-vol sensitivities of model prices (DESIGN.md §4.6).  The model ivol sigma(F, p) is defined by B(F, sigma) = P(F, p), B the
// discounted Black-76 price, P the model price, F the slice forward (sticky strike: it moves both P and Black's F), p the NP model
// parameters.  One thread per quote inverts the price with black_implied_vol -- the same function on the same doubles as
// b200sv_bsm_implied_vols and the fused batch pricers, so the ivols are bit-identical to theirs -- and applies the implicit-function rule
//   sigma_p  = P_p / B_s                                   sigma_F  = (P_F - B_F) / B_s
//   sigma_FF = (P_FF - B_FF - 2 B_Fs sigma_F - B_ss sigma_F^2) / B_s
//   sigma_Fp = (P_Fp - B_Fs sigma_p - B_ss sigma_F sigma_p) / B_s          (SECOND only)
//   sigma_pq = (P_pq - B_ss sigma_p sigma_q) / B_s                          (SECOND only)
// rows: [2 + NP][n] = (P_F, P_FF, P_p) then, when SECOND, vanna [NP][n] = P_Fp and hessian [NP(NP+1)/2][n] = P_pq (p <= q, row-major).
// out:  [n] ivols, then the sigma rows in the same layout.  Row-major [row][n], so a warp's loads and stores of one row are coalesced.
// Where the ivol is NaN every row is NaN.  Where it is an end of the inversion bracket (1e-8 or 10) the ivol does not move with the
// price and every row is 0: a calibration objective that still counts the quote then gets the gradient of what it counts.
template <int NP, bool SECOND>
__global__ void __launch_bounds__(64) black_ivol_sensitivities_kernel(const QuoteSpec* __restrict__ q, int n, const double* __restrict__ rows,
                                                                      double* __restrict__ out) {
  constexpr int NH = NP * (NP + 1) / 2;
  constexpr int NROWS = 2 + NP + (SECOND ? NP + NH : 0);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const QuoteSpec s = q[i];
  const double vol = black_implied_vol(s.forward, s.strike, s.ttm, s.discfactor, s.price, s.type);
  out[i] = vol;
  double* sig = out + n;
  if (vol != vol || black_vol_at_bracket_end(vol)) {
    const double fill = vol != vol ? vol : 0.0;
#pragma unroll 4
    for (int r = 0; r < NROWS; ++r) sig[(size_t)r * n + i] = fill;
    return;
  }
  const BlackPartials b = black_partials(s.forward, s.strike, s.ttm, s.discfactor, vol, s.type);
  const double sF = (rows[i] - b.dF) / b.vega;
  sig[i] = sF;
  sig[(size_t)n + i] = (rows[(size_t)n + i] - b.dFF - 2.0 * b.dFv * sF - b.dvv * sF * sF) / b.vega;
  double sp[NP];
#pragma unroll
  for (int k = 0; k < NP; ++k) {
    sp[k] = rows[(size_t)(2 + k) * n + i] / b.vega;
    sig[(size_t)(2 + k) * n + i] = sp[k];
  }
  if constexpr (SECOND) {
    const double cF = b.dFv + b.dvv * sF;
#pragma unroll
    for (int k = 0; k < NP; ++k) {
      const size_t r = (size_t)(2 + NP + k) * n + i;
      sig[r] = (rows[r] - cF * sp[k]) / b.vega;
    }
    int h = 2 + 2 * NP;
#pragma unroll
    for (int a = 0; a < NP; ++a)
#pragma unroll
      for (int c = a; c < NP; ++c, ++h) {
        const size_t r = (size_t)h * n + i;
        sig[r] = (rows[r] - b.dvv * sp[a] * sp[c]) / b.vega;
      }
  }
}

// Implied-vol theta (DESIGN.md §4.8): B(sigma, T) = P(T) at fixed F and D gives -d sigma / dT = (theta + B_T) / B_sigma with theta = -P_T
// and B_T = B_sigma sigma / (2 T) (Black-76 depends on T through sigma sqrt T only).  One thread per quote, the same inversion as
// black_ivol_kernel (bit-identical ivols) and the same NaN / bracket-end rules as the sensitivity rows.
__global__ void __launch_bounds__(64) black_ivol_theta_kernel(const QuoteSpec* __restrict__ q, int n, const double* __restrict__ theta,
                                                              double* __restrict__ ivols, double* __restrict__ ivol_theta) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const QuoteSpec s = q[i];
  const double vol = black_implied_vol(s.forward, s.strike, s.ttm, s.discfactor, s.price, s.type);
  ivols[i] = vol;
  if (vol != vol || black_vol_at_bracket_end(vol)) {
    ivol_theta[i] = vol != vol ? vol : 0.0;
    return;
  }
  const double vega = black_partials(s.forward, s.strike, s.ttm, s.discfactor, vol, s.type).vega;
  ivol_theta[i] = (theta[i] + vega * vol / (2.0 * s.ttm)) / vega;
}

constexpr int IVOL_SENS_MAX_NP = 15;     // the Hawkes parameter count, the largest of the Fourier chain pricers

template <int NP>
static int launch_ivol_sensitivities(int np, bool second, int n, const QuoteSpec* q, const double* rows, double* out, cudaStream_t st) {
  if constexpr (NP > IVOL_SENS_MAX_NP) {
    return fail(-1, "invalid argument: NP must be in 1..15");
  } else {
    if (np != NP) return launch_ivol_sensitivities<NP + 1>(np, second, n, q, rows, out, st);
    const int blocks = (n + 63) / 64;
    if (second) black_ivol_sensitivities_kernel<NP, true><<<blocks, 64, 0, st>>>(q, n, rows, out);
    else black_ivol_sensitivities_kernel<NP, false><<<blocks, 64, 0, st>>>(q, n, rows, out);
    return check_launch("black_ivol_sensitivities_kernel");
  }
}

}  // namespace b200sv

using namespace b200sv;

// one QuoteSpec per quote of the chain, flat in chain order; -3 on an unknown type code
static int quote_specs(int M, const double* ttms, const double* forwards, const double* discfactors, const int* offsets, const double* strikes,
                       const int8_t* types, const double* prices, std::vector<QuoteSpec>& q) {
  q.resize(offsets[M] - offsets[0]);
  for (int m = 0; m < M; ++m)
    for (int j = offsets[m]; j < offsets[m + 1]; ++j) {
      if (types[j] < 0 || types[j] > 3) return fail(-3, "unknown option payoff code");
      q[j - offsets[0]] = QuoteSpec{forwards[m], strikes[j], ttms[m], discfactors[m], prices[j - offsets[0]], (int)types[j]};
    }
  return 0;
}

static int bsm_implied_vols(int M, const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                            const double* strikes, const int8_t* types, const double* prices, double* ivols_out, int* iterations_out) {
  B200SV_REQUIRE(ttms && forwards && discfactors && offsets && strikes && types && prices && ivols_out, "null pointer");
  B200SV_REQUIRE(M >= 1, "M >= 1");
  const int n = offsets[M] - offsets[0];
  if (n <= 0) return 0;
  std::vector<QuoteSpec> q;
  if (int rc = quote_specs(M, ttms, forwards, discfactors, offsets, strikes, types, prices, q)) return rc;
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  DevBuf dq(st), dv(st), di(st);
  B200SV_CUDA(dq.alloc(sizeof(QuoteSpec) * n));
  B200SV_CUDA(dv.alloc(sizeof(double) * n));
  B200SV_CUDA(cudaMemcpyAsync(dq.p, q.data(), sizeof(QuoteSpec) * n, cudaMemcpyHostToDevice, st));
  if (iterations_out) {
    B200SV_CUDA(di.alloc(sizeof(int) * n));
    black_ivol_count_kernel<<<(n + 63) / 64, 64, 0, st>>>(dq.as<QuoteSpec>(), n, dv.as<double>(), di.as<int>());
    if (int rc = check_launch("black_ivol_count_kernel")) return rc;
    B200SV_CUDA(cudaMemcpyAsync(iterations_out, di.p, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
  } else {
    black_ivol_kernel<<<(n + 63) / 64, 64, 0, st>>>(dq.as<QuoteSpec>(), n, dv.as<double>());
    if (int rc = check_launch("black_ivol_kernel")) return rc;
  }
  B200SV_CUDA(cudaMemcpyAsync(ivols_out, dv.p, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
  return sync.done();
}

extern "C" int b200sv_bsm_implied_vols(int M, const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                       const double* strikes, const int8_t* types, const double* prices, double* ivols_out) {
  return bsm_implied_vols(M, ttms, forwards, discfactors, offsets, strikes, types, prices, ivols_out, nullptr);
}

extern "C" int b200sv_debug_bsm_implied_vols(int M, const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                             const double* strikes, const int8_t* types, const double* prices, double* ivols_out,
                                             int* iterations_out) {
  B200SV_REQUIRE(iterations_out, "null pointer");
  return bsm_implied_vols(M, ttms, forwards, discfactors, offsets, strikes, types, prices, ivols_out, iterations_out);
}

extern "C" int b200sv_bsm_implied_vol_sensitivities(int M, const double* ttms, const double* forwards, const double* discfactors,
                                                    const int* offsets, const double* strikes, const int8_t* types, const double* prices,
                                                    int NP, const double* greeks, const double* vanna, const double* hessian,
                                                    double* ivols_out, double* ivol_greeks_out, double* ivol_vanna_out,
                                                    double* ivol_hessian_out) {
  B200SV_REQUIRE(ttms && forwards && discfactors && offsets && strikes && types && prices && greeks && ivols_out && ivol_greeks_out,
                 "null pointer");
  B200SV_REQUIRE(M >= 1, "M >= 1");
  B200SV_REQUIRE(NP >= 1 && NP <= IVOL_SENS_MAX_NP, "NP must be in 1..15");
  B200SV_REQUIRE(!vanna == !hessian, "vanna and hessian are given together or not at all");
  B200SV_REQUIRE(!vanna == !ivol_vanna_out && !hessian == !ivol_hessian_out, "every second-order input needs its output and vice versa");
  const bool second = vanna != nullptr;
  const int n = offsets[M] - offsets[0];
  if (n <= 0) return 0;
  std::vector<QuoteSpec> q;
  if (int rc = quote_specs(M, ttms, forwards, discfactors, offsets, strikes, types, prices, q)) return rc;
  const size_t nh = (size_t)NP * (NP + 1) / 2, n1 = 2 + NP, nrows = n1 + (second ? NP + nh : 0);
  std::vector<double> rows(nrows * n);                      // the input rows packed as the kernel reads them: one upload
  std::memcpy(rows.data(), greeks, sizeof(double) * n1 * n);
  if (second) {
    std::memcpy(rows.data() + n1 * n, vanna, sizeof(double) * NP * n);
    std::memcpy(rows.data() + (n1 + NP) * n, hessian, sizeof(double) * nh * n);
  }
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  DevBuf dq(st), drows(st), dout(st);
  B200SV_CUDA(dq.upload(q.data(), n));
  B200SV_CUDA(drows.upload(rows.data(), rows.size()));
  B200SV_CUDA(dout.alloc(sizeof(double) * (1 + nrows) * n));
  if (int rc = launch_ivol_sensitivities<1>(NP, second, n, dq.as<QuoteSpec>(), drows.as<double>(), dout.as<double>(), st)) return rc;
  std::vector<double> out((1 + nrows) * n);
  B200SV_CUDA(dout.download(out.data(), out.size()));
  if (int rc = sync.done()) return rc;
  const double* o = out.data();
  std::memcpy(ivols_out, o, sizeof(double) * n);
  std::memcpy(ivol_greeks_out, o + n, sizeof(double) * n1 * n);
  if (second) {
    std::memcpy(ivol_vanna_out, o + (1 + n1) * n, sizeof(double) * NP * n);
    std::memcpy(ivol_hessian_out, o + (1 + n1 + NP) * n, sizeof(double) * nh * n);
  }
  return 0;
}

extern "C" int b200sv_bsm_implied_vol_theta(int M, const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                            const double* strikes, const int8_t* types, const double* prices, const double* theta,
                                            double* ivols_out, double* ivol_theta_out) {
  B200SV_REQUIRE(ttms && forwards && discfactors && offsets && strikes && types && prices && theta && ivols_out && ivol_theta_out,
                 "null pointer");
  B200SV_REQUIRE(M >= 1, "M >= 1");
  const int n = offsets[M] - offsets[0];
  if (n <= 0) return 0;
  std::vector<QuoteSpec> q;
  if (int rc = quote_specs(M, ttms, forwards, discfactors, offsets, strikes, types, prices, q)) return rc;
  cudaStream_t st = current_stream();
  ensure_pool_threshold();
  StreamSync sync(st);
  DevBuf dq(st), dth(st), dv(st), dt(st);
  B200SV_CUDA(dq.upload(q.data(), n));
  B200SV_CUDA(dth.upload(theta, n));
  B200SV_CUDA(dv.alloc(sizeof(double) * n));
  B200SV_CUDA(dt.alloc(sizeof(double) * n));
  black_ivol_theta_kernel<<<(n + 63) / 64, 64, 0, st>>>(dq.as<QuoteSpec>(), n, dth.as<double>(), dv.as<double>(), dt.as<double>());
  if (int rc = check_launch("black_ivol_theta_kernel")) return rc;
  B200SV_CUDA(dv.download(ivols_out, n));
  B200SV_CUDA(dt.download(ivol_theta_out, n));
  return sync.done();
}
