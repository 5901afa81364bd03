// black.cuh -- Black-76 implied volatility of one quote (shared by ivol_kernels.cu and the batched chain pricers of mgf_kernels.cu /
// the fused finalize kernels of mc_kernels.cu, so every inversion in the library is this one function).
//
// The quote is turned into the price q of its OUT-OF-THE-MONEY twin (the put for K < F, the call for K >= F) and the iteration solves
// that side's formula, K N(-d2) - F N(-d1) or F N(d1) - K N(d2), whose value keeps its relative precision however deep in the tail.
// Solving the call side for an out-of-the-money put instead (c = p + F - K) rounds p away against F - K: NaN below ~2e-17 F, vol
// errors up to 0.14 just above.  An in-the-money quote is brought to its twin by q = p / D - |F - K| with the exact remainder of the
// division (fma) and the exact error of F - K (two-sum), so the time value keeps its own precision too.
//
// Safeguarded Newton in total vol s = vol sqrt(T): start at the inflection point sqrt(2 |ln F/K|) (Brenner-Subrahmanyam at the money),
// keep the bracket [1e-8, 10] sqrt(T) updated by the sign of every residual.  Where the model price is above twice q the step is
// Newton's on ln(price) against ln(s): the tail price is exponential in 1/s^2 and the near-money price linear in s, so plain Newton
// would crawl down the one and overshoot below zero on the other.  A step that leaves the bracket moves 4x towards an end not yet
// tried, else to the bracket's geometric midpoint.  The rounding of d1 and d2 themselves is carried to first order (two-sum errors
// e1, e2; F phi(d1) = K phi(d2)), since at |d| ~ 9 it alone would cost d^2 ulp of each term.  Stop when the residual is within 4 ulp of
// the two terms (after one last Newton step) or the step / bracket is within 2 ulp of s.  On a grid of 3200 quotes (|ln(F/K)| / (vol
// sqrt T) <= 9, vol in [0.01, 5], T in [3e-4, 10]) the restatement oracle/bsm.py needs at most ~32 iterations, mean ~13; the cap is 64.
// Accuracy: |vol - vol*| <= A eps (F N(+-d1) + K N(+-d2) + q) / vega + 4 ulp, the backward error of the out-of-the-money formula
// (tests/test_gpu_ivol_edges.py, tests/test_bsm_oracle_edges.py).
// Quotes outside the strict no-arbitrage bounds (time value <= 0, p / D >= F for a call or >= K for a put, F, K, T or D <= 0,
// anything non-finite) give NaN; a root outside the bracket returns the bracket's nearer end, 1e-8 or 10 (to the rounding of s / sqrt T).
// `iterations` (debug only: b200sv_debug_bsm_implied_vols) receives the number of residual evaluations; the product passes nullptr.
#pragma once
#include <cmath>

#include "../../include/b200sv.h"

namespace b200sv {

__device__ __forceinline__ double black_call(double F, double K, double sdev) {
  const double d1 = log(F / K) / sdev + 0.5 * sdev;
  return F * normcdf(d1) - K * normcdf(d1 - sdev);
}

__device__ __forceinline__ double black_implied_vol(double forward, double strike, double ttm, double discfactor, double price, int type,
                                                    int* iterations = nullptr) {
  if (iterations) *iterations = 0;
  if (!(forward > 0.0 && strike > 0.0 && ttm > 0.0 && discfactor > 0.0) || !isfinite(forward) || !isfinite(strike) || !isfinite(ttm) ||
      !isfinite(discfactor) || !isfinite(price))
    return NAN;
  const bool is_call = (type == B200SV_CALL || type == B200SV_INV_CALL);
  const double r = price / discfactor;
  const double rr = fma(-r, discfactor, price) / discfactor;                  // p / D = r + rr
  const double room = fma(discfactor, is_call ? forward : strike, -price);    // sign of D F - p (call), D K - p (put): exact
  double q = r;                                                                // the out-of-the-money twin's undiscounted price
  if (is_call ? (strike < forward) : (strike > forward)) {                     // in the money: q = p / D - |F - K|
    const double hi = is_call ? forward : strike, lo = is_call ? strike : forward;
    const double d = hi - lo, bb = d - hi, t = (hi - (d - bb)) + (-lo - bb);   // |F - K| = d + t exactly
    q = (r - d) + (rr - t);
  }
  if (!(q > 0.0 && room > 0.0)) return NAN;
  const bool put_side = strike < forward;
  const double srt = sqrt(ttm);
  const double x = log(forward / strike);
  const double a0 = 1e-8 * srt, b0 = 10.0 * srt;
  double a = a0, b = b0;
  double s = sqrt(2.0 * fabs(x));
  if (!(s > a && s < b)) s = fmin(fmax(2.5066282746310002 * q / forward, 2.0 * a), 0.5 * b);   // at the money: Brenner-Subrahmanyam
  int it = 0;
  while (it < 64) {
    ++it;
    const double xs = x / s, hs = 0.5 * s;
    const double d1 = xs + hs, d2 = xs - hs;
    double bb = d1 - xs;
    const double e1 = (xs - (d1 - bb)) + (hs - bb);                            // d1 exact = d1 + e1 (given xs)
    bb = d2 - xs;
    const double e2 = (xs - (d2 - bb)) + (-hs - bb);
    const double t1 = put_side ? strike * normcdf(-d2) : forward * normcdf(d1);
    const double t2 = put_side ? forward * normcdf(-d1) : strike * normcdf(d2);
    const double vega = forward * 0.3989422804014327 * exp(-0.5 * d1 * d1);   // d price / d s
    const double f = (t1 - t2) + vega * (e1 - e2);
    if (fabs(f - q) <= 8.9e-16 * (t1 + t2) && vega > 0.0) {                   // within the noise of the formula: one last step
      s -= (f - q) / vega;
      break;
    }
    if (f < q) a = s; else b = s;
    double sn = f > 2.0 * q ? s * exp(-log(f / q) * f / (s * vega)) : s - (f - q) / vega;
    if (!(sn > a && sn < b))                                                   // also catches NaN / inf from a vanishing vega
      sn = (sn >= b && b == b0) ? fmin(4.0 * s, b) : (sn <= a && a == a0) ? fmax(0.25 * s, a) : sqrt(a * b);
    const double step = fabs(sn - s);
    s = sn;
    if (step <= 4.5e-16 * s || b - a <= 4.5e-16 * b) break;                   // within 2 ulp
  }
  if (iterations) *iterations = it;
  return s / srt;
}

// True where black_implied_vol returned an end of its bracket [1e-8, 10] (to the rounding of s / sqrt T, with a 1e-10 relative margin):
// the root lies outside it, so the returned vol does not move with the price.
__device__ __forceinline__ bool black_vol_at_bracket_end(double vol) {
  return vol <= 1e-8 * (1.0 + 1e-10) || vol >= 10.0 * (1.0 - 1e-10);
}

// Partial derivatives of the discounted Black-76 price B(F, vol) of one quote, in vol (not total vol): s = vol sqrt T,
// d1 = ln(F/K) / s + s / 2, d2 = d1 - s, n = phi(d1), D the discount factor.  Calls and puts differ only in B_F; IC / IP are priced as
// C / P, as in black_implied_vol.
struct BlackPartials {
  double vega;   // B_vol     = D F n sqrt T
  double dF;     // B_F       = D N(d1) (call), D (N(d1) - 1) (put)
  double dFF;    // B_FF      = D n / (F s)
  double dFv;    // B_F,vol   = -D n d2 / vol
  double dvv;    // B_vol,vol = B_vol d1 d2 / vol
};

__device__ __forceinline__ BlackPartials black_partials(double forward, double strike, double ttm, double discfactor, double vol, int type) {
  const bool is_call = (type == B200SV_CALL || type == B200SV_INV_CALL);
  const double srt = sqrt(ttm), s = vol * srt;
  const double d1 = log(forward / strike) / s + 0.5 * s, d2 = d1 - s;
  const double n = 0.3989422804014327 * exp(-0.5 * d1 * d1);
  BlackPartials b;
  b.vega = discfactor * forward * n * srt;
  b.dF = discfactor * (is_call ? normcdf(d1) : -normcdf(-d1));
  b.dFF = discfactor * n / (forward * s);
  b.dFv = -discfactor * n * d2 / vol;
  b.dvv = b.vega * d1 * d2 / vol;
  return b;
}

}  // namespace b200sv
