// gauss64.cuh -- fp64 Box-Muller for the fused MC kernels, written for the fp64-pipe-bound instruction mix (DESIGN.md 3.2).
//
// CUDA's libdevice log / sqrt / sincospi cost ~80 fp64-pipe instructions per pair of normals (the all-fp64 mode of round 1 ran 3.2x
// slower than the float-draw mode, VERDICT r1).  The fp64 pipe of an H100 SM issues one warp instruction every 2 clocks per
// sub-partition and is the resource the log-vol recursion already lives on, so the draw is rebuilt around three small shared-memory
// tables (the load/store unit is idle) and short polynomials:
//
//   R^2 = -2 ln(u1):  u1 = 2^e m, m in [sqrt(1/2), sqrt(2)) (fdlibm split, integer ops on the high word);  i = 7 leading bits of m;
//                     r = m * (1/c_i) - 1, |r| <= 3.9e-3;  -2 ln u1 = e (-2 ln 2) + (-2 ln c_i) - 2 log1p(r),  log1p to r^6 (next: 2e-18).
//                     The interval that contains m = 1 has c = 1 exactly: full relative accuracy as u1 -> 1.        8 fp64 + 1 I2F
//   R = sqrt(R^2):    y0 = rsqrt.approx.f64 (MUFU.RSQ64H), one third-order step  e = 1 - x y0^2,  R = x y0 (1 + e/2 + 3 e^2/8)   5 fp64
//   sin/cos(2 pi u2): j = 8 leading bits of u2 (table of sin/cos at the interval centres), f = u2 - centre, |2 pi f| <= 0.0123:
//                     sin to f^5, cos to f^6 (next terms 8e-18, 1e-20), angle addition.                               12 fp64
//   z0 = R cos, z1 = R sin                                                                                             2 fp64
// => 27 fp64-pipe instructions per pair instead of ~80.  Max error against 40-digit references on every table seam and at u1 = 2^-52
// (R = 8.49) and 1 - 2^-52: 1.89 x 2^-52 max(1, R) on the normals, an absolute error that grows with R (one ulp of R = 8.49 is 1.8e-15)
// (tests/test_gpu_mc_edges.py, H100).  Tables: 2 KB + 4 KB of shared memory per CTA (gauss64_table_init()).
#pragma once
#include <cstdint>

namespace b200sv {

#include "gauss64_tables.inc"

__shared__ double2 g_log_tab[128];
__shared__ double2 g_sincos_tab[256];

// call once per CTA before the first draw (ends with __syncthreads())
__device__ __forceinline__ void gauss64_table_init() {
  for (int i = threadIdx.x; i < 128; i += blockDim.x) g_log_tab[i] = make_double2(kLogTab[i][0], kLogTab[i][1]);
  for (int i = threadIdx.x; i < 256; i += blockDim.x) g_sincos_tab[i] = make_double2(kSinCosTab[i][0], kSinCosTab[i][1]);
  __syncthreads();
}

// -2 ln(u) for a positive normal double u <= 1 given as (hi, lo) words
__device__ __forceinline__ double neg2_log(uint32_t hi, uint32_t lo) {
  const uint32_t hx = hi + (0x3ff00000u - 0x3fe6a09eu);
  const int e = (int)(hx >> 20) - 0x3ff;
  const double m = __hiloint2double((int)((hx & 0x000fffffu) + 0x3fe6a09eu), (int)lo);
  const double2 T = g_log_tab[(hx >> 13) & 127u];
  const double r = fma(m, T.x, -1.0);
  double p = fma(r, 1.0 / 3.0, -2.0 / 5.0);     // -2 log1p(r) = r (-2 + r (1 + r (-2/3 + r (1/2 + r (-2/5 + r/3)))))
  p = fma(p, r, 0.5);
  p = fma(p, r, -2.0 / 3.0);
  p = fma(p, r, 1.0);
  p = fma(p, r, -2.0);
  const double t = fma((double)e, -1.3862943611198906188, T.y);
  return fma(r, p, t);
}

// sqrt(x) for x in [2^-60, 2^10]
__device__ __forceinline__ double fast_sqrt_pos(double x) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  const double t = x * y;
  const double e = fma(-t, y, 1.0);
  const double q = e * fma(e, 0.375, 0.5);
  return fma(t, q, t);
}

// sin / cos of 2 pi u2 where u2 = (j + mantissa-fraction) / 256:  j = interval index, (fhi, flo) = words of a double in [1, 1 + 2^-8)
// whose excess over 1 is the position inside the interval
__device__ __forceinline__ void sincos_turn(uint32_t j, uint32_t fhi, uint32_t flo, double& s, double& c) {
  const double f = __hiloint2double((int)fhi, (int)flo) - 1.001953125;   // position - half interval: [-2^-9, 2^-9)
  const double2 T = g_sincos_tab[j];
  const double w = f * f;
  // phi = 2 pi f
  double sp = fma(w, 81.605249276075054203, -41.341702240399760234);     // (2pi)^5/120, -(2pi)^3/6
  sp = fma(sp, w, 6.2831853071795864769);
  sp = sp * f;                                                           // sin(phi)
  double cp = fma(w, -85.456817206693725, 64.939394022668291491);        // -(2pi)^6/720, (2pi)^4/24
  cp = fma(cp, w, -19.739208802178717238);                               // -(2pi)^2/2
  cp = fma(cp, w, 1.0);                                                  // cos(phi)
  s = fma(T.x, cp, T.y * sp);
  c = fma(T.y, cp, -(T.x * sp));
}

// One pair of fp64 normals from a Philox block: 52-bit uniforms (the lowest bit of u1's mantissa is forced to 1 so that u1 < 1 and
// R > 0 always -- a 51-bit uniform).  u1 = 2 - d(r0, r1 | 1) in (0, 1),  u2 = d(r2, r3) - 1 in [0, 1),  d(hi, lo) = double with
// exponent 0x3FF and mantissa (hi >> 12):lo.   Z0 = R cos(2 pi u2), Z1 = R sin(2 pi u2), R = sqrt(-2 ln u1).
__device__ __forceinline__ void box_muller_f64_fast(uint4 r, double& z0, double& z1) {
  const double u1 = 2.0 - __hiloint2double((int)(0x3FF00000u | (r.x >> 12)), (int)(r.y | 1u));
  const double rad = fast_sqrt_pos(neg2_log((uint32_t)__double2hiint(u1), (uint32_t)__double2loint(u1)));
  double s, c;
  sincos_turn(r.z >> 24, 0x3FF00000u | ((r.z >> 12) & 0xFFFu), r.w, s, c);
  z0 = rad * c;
  z1 = rad * s;
}

// The SAME uniforms as the float Box-Muller of philox.cuh (u1 = (ra + 1/2) 2^-32, angle = rb 2^-32 turns), evaluated in fp64:
// the "paired" check mode B200SV_GAUSS_F64_PAIRED -- differences against the default mode isolate the SFU approximation error.
__device__ __forceinline__ void box_muller_f64_u32(uint32_t ra, uint32_t rb, double& z0, double& z1) {
  const double u1 = fma((double)ra, 2.3283064365386963e-10, 1.1641532182693481e-10);
  const double rad = fast_sqrt_pos(neg2_log((uint32_t)__double2hiint(u1), (uint32_t)__double2loint(u1)));
  double s, c;
  sincos_turn(rb >> 24, 0x3FF00000u | ((rb >> 12) & 0xFFFu), rb << 20, s, c);
  z0 = rad * c;
  z1 = rad * s;
}

}  // namespace b200sv
