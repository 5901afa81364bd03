/* b200sv.h -- C ABI of libb200sv.so: the H100 (sm_90a) replacement for the two numerical hot paths of
 * ArturSepp/StochVolModels (stochvolmodels 2.2.0).  Plain pointers and sizes; no torch / C++ types.
 *
 * Each entry point names the reference interface it replaces (paths relative to
 * src/stochvolmodels of the reference).  The reference is pure Python + Numba, so "the FFI for this path" is a
 * ctypes binding: INTEGRATION.md shows the stub a maintainer adds inside LogSVPricer / HestonPricer.
 *
 * Conventions
 *   - return 0 on success, <0 on error; b200sv_last_error() returns a thread-local message.
 *   - arrays are caller-owned; no pointer is retained after return.
 *   - "host-level" calls (no _dev_ in the name) take HOST pointers, run on the current CUDA device, and are
 *     synchronous: H2D copies of the inputs and D2H copies of the results happen inside the call.
 *   - "device-level" calls (b200sv_dev_*) take DEVICE pointers and a cudaStream_t (as void*; NULL = the legacy
 *     default stream), enqueue work and return without synchronising.  They are what a multi-GPU host composes with
 *     its own collectives (two tiny all-reduces per maturity, see DESIGN.md "multi-GPU").
 *   - option chain layout ("CSR"): strikes[offsets[m] .. offsets[m+1]) belong to maturity m;
 *     types[] uses B200SV_CALL.. codes in the same positions.
 *   - all floating point crossing the ABI is IEEE float64, as in the reference.
 */
#ifndef B200SV_H
#define B200SV_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200SV_VERSION 100 /* 0.1.0 */

/* option payoff codes: utils/config.py:8-14 OptionType {'C','P','IC','IP'} */
enum { B200SV_CALL = 0, B200SV_PUT = 1, B200SV_INV_CALL = 2, B200SV_INV_PUT = 3 };
/* utils/config.py:17-24 VariableType */
enum { B200SV_LOG_RETURN = 1, B200SV_Q_VAR = 2, B200SV_SIGMA = 3 };
/* pricers/logsv/affine_expansion.py:43-54 ExpansionOrder */
enum { B200SV_ORDER_FIRST = 1, B200SV_ORDER_SECOND = 2 };

/* MC arithmetic flags (bit-or).  Default 0 = fp64 state arithmetic, Gaussians drawn by a float Box-Muller on the SFU
 * and widened (the draws are random inputs, not reference arithmetic).  B200SV_GAUSS_F64 draws them in fp64 as well;
 * B200SV_STATE_F32 keeps x / log-sigma / qvar in float registers (payoff moments stay fp64). */
enum { B200SV_STATE_F64 = 0, B200SV_STATE_F32 = 1, B200SV_GAUSS_F32 = 0, B200SV_GAUSS_F64 = 2,
       /* check mode: the DEFAULT stream's 32-bit uniforms pushed through the fp64 Box-Muller (paired with the default mode path by path,
        * so that price differences isolate the SFU approximation error of the float draws; tests/test_gpu_gauss_bias.py) */
       B200SV_GAUSS_F64_PAIRED = 4 };
/* Heston variance scheme: 0 = the reference's floor-Euler (pricers/heston_pricer.py:369-379, v = max(v, 1e-4)); 1 = opt-in Andersen (2008)
 * quadratic-exponential scheme with central discretisation (BASELINE.json config 2 names it; the reference does not have it) */
enum { B200SV_HESTON_EULER_FLOOR = 0, B200SV_HESTON_QE = 1 };

/* pricers/logsv/logsv_params.py:35-83 LogSvParams (the six model floats; kappa2=None already mapped to kappa1/theta) */
typedef struct {
  double sigma0, theta, kappa1, kappa2, beta, volvol;
} b200sv_logsv_params;

/* pricers/heston_pricer.py:27-41 HestonParams */
typedef struct {
  double v0, theta, kappa, rho, volvol;
} b200sv_heston_params;

/* pricers/hawkes_jd_pricer.py:41-65 HawkesJDParams (the sixteen model floats, in the order of the dataclass with lambda_p / lambda_m moved next
 * to their intensities' parameters as listed here) */
typedef struct {
  double mu, sigma, shift_p, mean_p, shift_m, mean_m;
  double lambda_p, theta_p, kappa_p, beta1_p, beta2_p;
  double lambda_m, theta_m, kappa_m, beta1_m, beta2_m;
} b200sv_hawkes_params;

const char* b200sv_last_error(void);
/* CUDA stream (cudaStream_t as void*) on which the calling thread's HOST-LEVEL calls enqueue their copies and kernels and on which they
 * synchronise before returning; NULL (the default) = the legacy default stream.  Thread-local, like the error string: calls from different
 * threads on different streams run concurrently.  (SURVEY.md 8b asked for a stream on every call; the device-level b200sv_dev_* calls take it
 * as an argument, the host-level ones -- what a ctypes / cgo / JNI binding of the reference's functions binds -- take it from here so that
 * their signatures stay the reference's argument lists.) */
int b200sv_set_stream(void* stream);
void* b200sv_get_stream(void);
int b200sv_version(void);
/* number of this library's kernels launched by the calling thread since the last reset (bench "gpu_launches") */
long long b200sv_launch_count(void);
void b200sv_reset_launch_count(void);

/* ------------------------------------------------------------------------------------------------------------------
 * Monte Carlo, host-level
 * ------------------------------------------------------------------------------------------------------------------ */

/* replaces logsv_mc_chain_pricer (pricers/logsv_pricer.py:806-867) = chain loop over
 * simulate_logsv_x_vol_terminal (:950-1047) + compute_mc_vars_payoff (utils/mc_payoffs.py:10-88).
 * nb_steps_per_year follows set_time_grid (utils/funcs.py:24-47): S_m = int((ttm_m - ttm_{m-1}) * n) + 1.
 * Single-GPU, synchronous.  etas may be NULL (all 1).  prices_out, stderr_out: offsets[M]-offsets[0] doubles each. */
int b200sv_logsv_mc_chain(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                          const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                          const int8_t* types, long long nb_path, int nb_steps_per_year, int is_spot_measure,
                          int variable_type, uint64_t seed, int flags, double* prices_out, double* stderr_out);

/* replaces heston_mc_chain_pricer (pricers/heston_pricer.py:285-331) + simulate_heston_x_vol_terminal (:334-381).
 * nb_steps_per_year: the reference hard-wires 360 (:344). */
int b200sv_heston_mc_chain(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                           const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                           long long nb_path, int nb_steps_per_year, int variable_type, uint64_t seed, int flags,
                           int scheme, double* prices_out, double* stderr_out);

/* B parameter sets through the fused chain Monte Carlo in ONE call, all on the SAME Philox seed (common random numbers): the objective of
 * CalibrationEngine.MC (pricers/logsv_pricer.py:251-266 -- there: pre-drawn fixed normals W0s/W1s re-used across optimizer iterations;
 * here the counter-based generator re-draws the identical normals for every set, so nothing is stored or streamed).  params[B],
 * etas[B*M] (NULL = 1); prices_out / stderr_out / ivols_out are [B][J] in chain order (ivols_out may be NULL; Black-76 inversion fused into
 * the finalisation kernel).  LOG_RETURN payoffs.  Row b equals b200sv_logsv_mc_chain(params[b], seed) bit for bit. */
int b200sv_logsv_mc_chain_batch(const b200sv_logsv_params* params, int B, int M, const double* ttms, const double* forwards,
                                const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                const int8_t* types, long long nb_path, int nb_steps_per_year, int is_spot_measure, uint64_t seed,
                                int flags, double* prices_out, double* stderr_out, double* ivols_out);
int b200sv_heston_mc_chain_batch(const b200sv_heston_params* params, int B, int M, const double* ttms, const double* forwards,
                                 const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                 long long nb_path, int nb_steps_per_year, uint64_t seed, int flags, int scheme, double* prices_out,
                                 double* stderr_out, double* ivols_out);

/* Pathwise (forward-mode) Monte Carlo sensitivities of the chain pricers, in one pass (DESIGN.md §3.9).  Same arguments as
 * b200sv_logsv_mc_chain / b200sv_heston_mc_chain, same prices and std errors; in addition greeks_out and greeks_se_out, each
 * [1 + P][J] in chain order (J = offsets[M]-offsets[0]): row 0 = the forward delta d price / d forwards[m] of every strike of maturity m,
 * then one row per model parameter in struct field order --
 *   LogSV  (P = 6): sigma0, theta, kappa1, kappa2, beta, volvol   (kappa2 is held fixed when kappa1 or theta moves)
 *   Heston (P = 5): v0, theta, kappa, rho, volvol
 * greeks_se_out = discfactor * std(pathwise derivative) / sqrt(nb_path), the price's convention.  etas and discount factors are inputs,
 * not differentiated.  Unbiased for the discretised scheme.  flags: fp64 state with B200SV_GAUSS_F32 or B200SV_GAUSS_F64; Heston takes
 * scheme = B200SV_HESTON_EULER_FLOOR only.  Anything else returns an error.  Single GPU, synchronous. */
int b200sv_logsv_mc_chain_greeks(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                 const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                 const int8_t* types, long long nb_path, int nb_steps_per_year, int is_spot_measure, int variable_type,
                                 uint64_t seed, int flags, double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out);
int b200sv_heston_mc_chain_greeks(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                  const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                  long long nb_path, int nb_steps_per_year, int variable_type, uint64_t seed, int flags, int scheme,
                                  double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out);
/* The two calls above plus the Monte Carlo gamma d^2 price / d forwards[m]^2 of every strike, by conditional smoothing of the log-spot's
 * last step (DESIGN.md §3.9): gamma_out and gamma_se_out [J], the standard error with the greeks' convention.  Unbiased for the
 * discretised scheme at the given nb_path.  Every other output is bit-identical to the _greeks call with the same arguments; the same
 * flags and schemes are rejected.  Optional test hook (laststep_out may be NULL): laststep_out [M][2][n_paths_out] = (s, mu) of paths
 * [0, n_paths_out) after maturity m, where the last step is x = mu + s z0 given the state before it. */
int b200sv_logsv_mc_chain_greeks_gamma(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                       const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                       const int8_t* types, long long nb_path, int nb_steps_per_year, int is_spot_measure, int variable_type,
                                       uint64_t seed, int flags, double* prices_out, double* stderr_out, double* greeks_out,
                                       double* greeks_se_out, double* gamma_out, double* gamma_se_out, long long n_paths_out,
                                       double* laststep_out);
int b200sv_heston_mc_chain_greeks_gamma(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                        const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                        long long nb_path, int nb_steps_per_year, int variable_type, uint64_t seed, int flags, int scheme,
                                        double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out, double* gamma_out,
                                        double* gamma_se_out, long long n_paths_out, double* laststep_out);
/* The _greeks_gamma calls above (gamma_out == NULL: no gamma, and none of its launches) plus the Monte Carlo theta -d price / d ttms[m] of
 * every strike (DESIGN.md §3.12): theta_out and theta_se_out [J], per year, the standard error with the greeks' convention.  Pathwise in
 * the step length of maturity m's slice with its step count int((ttms[m] - ttms[m-1]) * nb_steps_per_year) + 1 held, and with the slice's
 * forward, discount factor and vol backbone eta and the earlier maturities held: unbiased for the discretised scheme.  Every other output is
 * bit-identical to the _greeks / _greeks_gamma call with the same arguments; the same flags and schemes are rejected.  Optional test hook
 * (dtheta_out may be NULL): dtheta_out [M][2][n_paths_out] = (dx, dq) / d dt of paths [0, n_paths_out) after maturity m, dt the slice's
 * step length. */
int b200sv_logsv_mc_chain_greeks_theta(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                       const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                       const int8_t* types, long long nb_path, int nb_steps_per_year, int is_spot_measure, int variable_type,
                                       uint64_t seed, int flags, double* prices_out, double* stderr_out, double* greeks_out,
                                       double* greeks_se_out, double* gamma_out, double* gamma_se_out, long long n_paths_out,
                                       double* laststep_out, double* theta_out, double* theta_se_out, double* dtheta_out);
int b200sv_heston_mc_chain_greeks_theta(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                        const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                        long long nb_path, int nb_steps_per_year, int variable_type, uint64_t seed, int flags, int scheme,
                                        double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out, double* gamma_out,
                                        double* gamma_se_out, long long n_paths_out, double* laststep_out, double* theta_out,
                                        double* theta_se_out, double* dtheta_out);

/* test entry points of the tangent stepper: one slice of ttm from (0, sigma0 | v0, 0) for the global paths [path_offset, path_offset + nb_path)
 * of Philox slice `slice_index`.  x, sigma | var, qvar: nb_path doubles; dx, dsigma | dvar, dqvar: [P][nb_path] tangents in the parameter
 * order above (host, out).  The state is the one b200sv_logsv_terminal / b200sv_heston_terminal compute. */
int b200sv_logsv_tangent_terminal(const b200sv_logsv_params* params, double ttm, long long nb_path, int nb_steps_per_year, int is_spot_measure,
                                  double eta, uint64_t seed, int flags, int slice_index, long long path_offset, double* x, double* sigma,
                                  double* qvar, double* dx, double* dsigma, double* dqvar);
int b200sv_heston_tangent_terminal(const b200sv_heston_params* params, double ttm, long long nb_path, int nb_steps_per_year, uint64_t seed,
                                   int flags, int slice_index, long long path_offset, double* x, double* var, double* qvar, double* dx,
                                   double* dvar, double* dqvar);

/* replaces LogSVPricer.simulate_terminal_values (pricers/logsv_pricer.py:590-611) -> simulate_logsv_x_vol_terminal.
 * x, sigma, qvar: nb_path doubles each (host, out). */
int b200sv_logsv_terminal(const b200sv_logsv_params* params, double ttm, long long nb_path, int nb_steps_per_year,
                          int is_spot_measure, double eta, uint64_t seed, int flags, double* x, double* sigma,
                          double* qvar);

/* replaces HestonPricer.simulate_terminal_values (pricers/heston_pricer.py:90-108). */
/* the same with PER-PATH initial arrays (pricers/logsv_pricer.py:1007-1020 accepts length-nb_path x0 / sigma0 / qvar0): in/out host arrays;
 * slice_index = Philox sub-stream (0 for a fresh start; m for the m-th consecutive call on one seed, as the chain pricer numbers its slices) */
int b200sv_logsv_terminal_from_state(const b200sv_logsv_params* params, double ttm, long long nb_path, int nb_steps_per_year, int is_spot_measure,
                                     double eta, uint64_t seed, int flags, int slice_index, double* x_inout, double* sigma_inout,
                                     double* qvar_inout);
int b200sv_heston_terminal(const b200sv_heston_params* params, double ttm, long long nb_path, int nb_steps_per_year,
                           uint64_t seed, int flags, int scheme, double* x, double* var, double* qvar);

/* replaces simulate_logsv_x_vol_terminal called with W0, W1, dt (pricers/logsv_pricer.py:1027-1047), the stepping
 * inside logsv_mc_chain_pricer_fixed_randoms (:1100-1162).  W0, W1: unit normals, row-major [S][N] (scaled by
 * sqrt(dt) inside, :1028-1030).  x, sigma, qvar: N doubles, updated in place.  Strict fp64, no FMA contraction,
 * reference evaluation order. */
int b200sv_logsv_step_fixed(double* x, double* sigma, double* qvar, const double* W0, const double* W1, int S,
                            long long N, double dt, const b200sv_logsv_params* params, double eta, int is_spot_measure);

/* Heston twin of the above (loop body pricers/heston_pricer.py:372-379). */
int b200sv_heston_step_fixed(double* x, double* var, double* qvar, const double* W0, const double* W1, int S,
                             long long N, double dt, const b200sv_heston_params* params);

/* replaces simulate_vol_paths (pricers/logsv_pricer.py:870-947; LogSVPricer.simulate_vol_paths :561-587): the whole volatility
 * path matrix sigma_t_out[(S+1)][nb_path] (row 0 = sigma0), S = int(ttm*n)+1.  brownians: optional host array [S][nb_path] of
 * SCALED increments (the reference's `brownians`); NULL draws sqrt(dt)*Z from the device Philox stream.  Strict fp64. */
int b200sv_logsv_vol_paths(const b200sv_logsv_params* params, double ttm, long long nb_path, int nb_steps_per_year,
                           int is_spot_measure, uint64_t seed, const double* brownians, double* sigma_t_out);

/* replaces compute_mc_vars_payoff (utils/mc_payoffs.py:10-88): forward re-centring with the nan-mean over all paths,
 * per-strike discounted nan-mean and nan-std/sqrt(N).  qvar may be NULL for B200SV_LOG_RETURN. */
int b200sv_mc_payoffs(const double* x, const double* qvar, long long N, double ttm, double forward, const double* strikes,
                      const int8_t* types, int J, double discfactor, int variable_type, double* prices_out,
                      double* stderr_out);

/* parity/debug export of the device RNG stream (csrc/philox.cuh): unit normals of paths [path0, path0+n) for chain
 * slice `slice`, steps 0..nsteps-1; z0, z1 row-major [nsteps][n] host doubles. */
int b200sv_device_normals(uint64_t seed, long long path0, long long n, int slice, int nsteps, int flags, double* z0,
                          double* z1);

/* ------------------------------------------------------------------------------------------------------------------
 * Monte Carlo, device-level building blocks (multi-GPU hosts put their all-reduces between them)
 * ------------------------------------------------------------------------------------------------------------------ */

/* one maturity slice of the fused stepper for local paths [0, n_local) whose global ids start at path_offset.
 * state arrays are float64 (B200SV_STATE_F64) or float32 (B200SV_STATE_F32) device arrays of n_local elements;
 * init != 0: start from (0, v_init, 0) instead of loading.  moments_out[2] (device) receives
 * (sum over non-NaN paths of forward*exp(x), count of non-NaN paths) for THIS rank. */
int b200sv_dev_logsv_slice(void* x, void* sigma, void* qvar, long long n_local, long long path_offset, int init,
                           const b200sv_logsv_params* params, double eta, int is_spot_measure, int nsteps, double dt,
                           int slice_index, double forward, uint64_t seed, int flags, double* moments_out, void* p2p_ctx,
                           void* stream);
int b200sv_dev_heston_slice(void* x, void* var, void* qvar, long long n_local, long long path_offset, int init,
                            const b200sv_heston_params* params, int nsteps, double dt, int slice_index, double forward,
                            uint64_t seed, int flags, int scheme, double* moments_out, void* p2p_ctx, void* stream);

/* per-strike payoff sums for local paths given the GLOBAL (all-reduced) re-centring moments[2]:
 * sums_out[3*J] (device) = (sum pay, sum pay^2, count non-NaN) per strike for THIS rank.
 * strikes / types are DEVICE arrays of J entries.  payoff_kinds_hint: what the HOST knows about types[] -- bit 0: some
 * 'C'/'P', bit 1: some 'IC'/'IP'; 1 selects the branch-free vanilla kernel, anything else (0 = unknown) the general one. */
int b200sv_dev_payoff_sums(const void* x, const void* qvar, long long n_local, int flags, double ttm, double forward,
                           const double* strikes, const int8_t* types, int J, int variable_type, int payoff_kinds_hint,
                           const double* moments, double* sums_out, void* p2p_ctx, void* stream);

/* turn GLOBAL sums[3*J] into prices / std errors (device arrays of J): price = df*s1/n, se = df*sqrt(s2/n-(s1/n)^2)/sqrt(N). */
int b200sv_dev_payoff_finalize(const double* sums, int J, double discfactor, long long total_paths, double* prices_out,
                               double* stderr_out, void* p2p_ctx, void* stream);

/* Peer-memory exchange of the two per-maturity messages (csrc/p2p.cuh): with a non-NULL p2p_ctx the calls above fuse the exchange into
 * their kernels instead of leaving it to the host's collective -- *_slice and *_payoff_sums PUBLISH their local values into every
 * peer's mailbox over NVLink from the reduction kernel that produces them, *_payoff_sums and *_payoff_finalize GATHER the global values
 * (summed in rank order) in their prologue; `moments` / `sums` arguments then carry this rank's local values only.  All ranks must
 * issue the same sequence of calls (a publish whose predecessor was never gathered on this rank gets a flag-wait inserted, which keeps
 * the double-buffered mailbox race-free when a maturity has no strikes or a rank has no paths).  create: allocates this rank's mailbox (max_values >= 3 * max strikes per slice) and returns a
 * 64-byte CUDA IPC handle to all-gather among the ranks of the node; connect: maps the peers' mailboxes (handles in rank order). */
int b200sv_p2p_create(int world, int rank, int max_values, void** ctx_out, unsigned char* handle_out);
int b200sv_p2p_connect(void* p2p_ctx, const unsigned char* handles);
int b200sv_p2p_destroy(void* p2p_ctx);
/* A gather that waits longer than the spin limit (default 2^24 polls of ~200 ns, ~3 s) poisons its value with NaN and sets bit r (the
 * peer that never published) of the context's status word.  b200sv_p2p_status synchronises `stream`, returns the word and clears it: a
 * host must call it after the chain's copy back and treat non-zero as an error (multi_gpu.mc_chain_distributed raises P2pTimeout). */
int b200sv_p2p_set_spin_limit(void* p2p_ctx, unsigned int spins);
int b200sv_p2p_status(void* p2p_ctx, unsigned int* status_out, void* stream);
/* test hook: pretend a publish was issued that never arrives, so that the next gather runs into the spin limit */
int b200sv_debug_p2p_lose_publish(void* p2p_ctx);
/* standalone halves of an exchange (ranks without local paths; tests): publish K local values / gather the K global ones */
int b200sv_dev_p2p_publish(void* p2p_ctx, const double* vals, int K, void* stream);
int b200sv_dev_p2p_gather(void* p2p_ctx, int K, double* out, void* stream);

/* device-level twins of b200sv_logsv_step_fixed / b200sv_heston_step_fixed (all arrays on the device; W row-major [S][N]):
 * the calibration inner loop logsv_mc_chain_pricer_fixed_randoms (pricers/logsv_pricer.py:1100-1162) keeps W0s/W1s
 * resident in HBM across optimizer iterations and calls these per maturity.  fast != 0 selects the throughput variant of the
 * LogSV stepper (the fused kernel's per-step update: folded constants, FMA, shared-polynomial exp pair; agrees with the strict
 * kernel to ~1e-14), whose bound is the 16 B/path-step HBM stream of normals. */
int b200sv_dev_logsv_step_fixed(double* x, double* sigma, double* qvar, const double* W0, const double* W1, int S,
                                long long N, double dt, const b200sv_logsv_params* params, double eta,
                                int is_spot_measure, int fast, void* stream);
int b200sv_dev_heston_step_fixed(double* x, double* var, double* qvar, const double* W0, const double* W1, int S,
                                 long long N, double dt, const b200sv_heston_params* params, void* stream);

/* Pathwise sensitivities of the LogSV chain on fixed unit normals resident on the device (DESIGN.md §4.7): W0s[m], W1s[m] are device
 * arrays [nsteps[m]][N] (row-major) of maturity m, stepped with dts[m] by the fast stepper above.  The chain block (ttms ... types, etas
 * [M] or NULL for ones) is on the HOST, as for the host-level chain calls.  Outputs are DEVICE arrays: prices_out, stderr_out [J_total]
 * bit-identical to b200sv_dev_logsv_step_fixed(fast = 1) + b200sv_dev_spot_moments + b200sv_dev_payoff_sums + b200sv_dev_payoff_finalize
 * on the same normals, parameters, etas and measure, and greeks_out / greeks_se_out [1 + 6][J_total]: row 0 the forward delta, then
 * d price / d (sigma0, theta, kappa1, kappa2, beta, volvol) in struct field order, with standard errors discfactor * std(g) / sqrt(N).
 * Asynchronous on `stream`. */
int b200sv_dev_logsv_mc_chain_greeks_fixed(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                           const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                           const int8_t* types, const double* const* W0s, const double* const* W1s, const int* nsteps,
                                           const double* dts, long long N, int is_spot_measure, int variable_type, double* prices_out,
                                           double* stderr_out, double* greeks_out, double* greeks_se_out, void* stream);

/* Rough-LogSV multi-factor Monte Carlo chain (Markovian lift of the rough kernel, 1 <= n_factors <= 8):
 * rough_logsv_mc_chain_pricer_fixed_randoms (pricers/logsv_pricer.py:1164-1232) -> log_spot_full_combined
 * (pricers/rough_logsv/split_simulation.py:466-479, f64 branch :340-361).  params[b].volvol carries the ORTHOGONAL vol-of-vol of set b
 * (the reference's `orthog_vol`); weights / nodes are [B][n_factors].  Every maturity m restarts at t = 0 and runs nsteps[m] steps of size
 * hs[m] (the reference's per-maturity `timegrids`), consuming rows [0, nsteps[m]) of the unit normals Z0 / Z1 (host, row-major
 * [z_rows][nb_path]); Z0 == Z1 == NULL draws them in-kernel from the Philox stream of csrc/philox.cuh (seed, flags = B200SV_GAUSS_*).
 * Outputs [B][J_total]: prices, "std errors" exactly as the reference returns them on this route -- discfactor * nanstd(payoff), NOT
 * divided by sqrt(nb_path) (it calls compute_mc_vars_payoff with (1, nb_path) arrays, utils/mc_payoffs.py:88) -- and optionally Black
 * implied vols (ivols_out may be NULL).  states_out (B == 1, may be NULL): [M][n_factors + 2][nb_path] = log-spot, factor values, quadratic
 * variance at each maturity. */
int b200sv_rough_logsv_mc_chain(const b200sv_logsv_params* params, int B, int n_factors, const double* weights, const double* nodes, int M,
                                const double* ttms, const double* forwards, const double* discfactors, const int* offsets, const double* strikes,
                                const int8_t* types, long long nb_path, const int* nsteps, const double* hs, const double* Z0, const double* Z1,
                                long long z_rows, int variable_type, uint64_t seed, int flags, double* prices_out, double* stderr_out,
                                double* ivols_out, double* states_out);

/* The rough chain above for ONE parameter set, plus pathwise sensitivities in the same pass (DESIGN.md §3.10): prices and "std errors"
 * as b200sv_rough_logsv_mc_chain on the same normals (discfactor * nanstd(payoff)), and greeks_out / greeks_se_out [1 + 6][J_total]: row 0
 * the forward delta, then d price / d (sigma0, theta, kappa1, kappa2, beta, volvol) in struct field order (volvol = the orthogonal
 * vol-of-vol), with real standard errors discfactor * std(g) / sqrt(nb_path).  weights / nodes [n_factors] are inputs, not differentiated.
 * Optional (may be NULL): states_out [M][n_factors + 2][nb_path] as above, tangents_out [M][6][n_factors + 2][nb_path] = the same rows
 * differentiated per parameter, resets_out [M] = the number of paths that took the reset-to-1e-6 branch at any step of maturity m's grid
 * (the pathwise rows omit the mass such paths move across that switch).  fp64 state only (B200SV_STATE_F32 is rejected); synchronous on
 * the library stream. */
int b200sv_rough_logsv_mc_chain_greeks(const b200sv_logsv_params* params, int n_factors, const double* weights, const double* nodes, int M,
                                       const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                       const double* strikes, const int8_t* types, long long nb_path, const int* nsteps, const double* hs,
                                       const double* Z0, const double* Z1, long long z_rows, int variable_type, uint64_t seed, int flags,
                                       double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out, double* states_out,
                                       double* tangents_out, double* resets_out);
/* The call above plus the Monte Carlo theta -d price / d ttms[m] of every strike (DESIGN.md §3.12): theta_out and theta_se_out [J], per year,
 * the standard error df std / sqrt(nb_path).  Every maturity restarts at t = 0 on its grid of nsteps[m] steps of hs[m]; theta is pathwise in
 * that step length with nsteps[m] held (d / d ttms[m] = (1 / nsteps[m]) d / d h), with the forward and discount factor held; the theta row
 * omits the same reset-branch mass as the parameter rows (resets_out).  Every other output is bit-identical to the _greeks call with the same
 * arguments.  Optional test hook (dtheta_out may be NULL): dtheta_out [M][2][n_paths_out] = (d log_spot, d qv) / d h of paths
 * [0, n_paths_out) at maturity m. */
int b200sv_rough_logsv_mc_chain_greeks_theta(const b200sv_logsv_params* params, int n_factors, const double* weights, const double* nodes, int M,
                                             const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                             const double* strikes, const int8_t* types, long long nb_path, const int* nsteps, const double* hs,
                                             const double* Z0, const double* Z1, long long z_rows, int variable_type, uint64_t seed, int flags,
                                             double* prices_out, double* stderr_out, double* greeks_out, double* greeks_se_out, double* states_out,
                                             double* tangents_out, double* resets_out, double* theta_out, double* theta_se_out,
                                             long long n_paths_out, double* dtheta_out);

/* Hawkes jump-diffusion Monte Carlo (pricers/hawkes_jd_pricer.py): 1800 steps per year (:752), state (x, lambda_p, lambda_m).
 * b200sv_hawkesjd_mc_chain   = hawkesjd_mc_chain_pricer (:644-715): chained slices, forward-recentred payoffs on x; in-kernel draws (Philox;
 *                              flags = B200SV_GAUSS_* for the normals, the jump clocks and sizes come from 32-bit uniforms through fp64 logs).
 * b200sv_hawkesjd_terminal   = simulate_hawkesjd_terminal (:718-779) with in-kernel draws; use_initial_arrays != 0: the three host arrays hold the
 *                              per-path initial state (in/out), else every path starts from (0, lambda_p, lambda_m) and the arrays are outputs.
 * b200sv_hawkesjd_step_fixed = the same update on caller-supplied inputs in the reference's own form, row-major [S][N] host arrays:
 *                              W0 = sqrt(dt) z, U_P / U_M = -ln(U)/dt, J_P / J_M = shift +- mean Exp(1) (:753-757) -- reference evaluation order,
 *                              no FMA contraction (parity entry).
 * b200sv_hawkesjd_device_draws exports, in that same form, what the in-kernel generator draws for paths [path0, path0 + n) of a slice. */
int b200sv_hawkesjd_mc_chain(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards, const double* discfactors,
                             const int* offsets, const double* strikes, const int8_t* types, long long nb_path, int variable_type, uint64_t seed,
                             int flags, double* prices_out, double* stderr_out);
/* b200sv_hawkesjd_mc_chain with Monte Carlo sensitivities (DESIGN.md §3.11): arguments as b200sv_hawkesjd_mc_chain, then
 * greeks_out / greeks_se_out [1 + 15][J]: the forward delta, then d price / d parameter in the order sigma, shift_p, mean_p, shift_m, mean_m,
 * lambda_p, theta_p, kappa_p, beta1_p, beta2_p, lambda_m, theta_m, kappa_m, beta1_m, beta2_m, each with its standard error df std(g) / sqrt(N).
 * Pathwise through the diffusion, the jump sizes and the intensities with the firing decisions frozen, plus the likelihood-ratio score of
 * the decisions; unbiased for the discretised scheme.  prices_out / stderr_out are bit-identical to b200sv_hawkesjd_mc_chain on the same
 * nb_path, seed and flags.  LOG_RETURN only (Q_VAR returns -4), fp64 state, B200SV_GAUSS_F32 or B200SV_GAUSS_F64, mean_p != 0 and
 * mean_m != 0 (dJ/dmean = (J - shift)/mean).
 * Optional per-path outputs for paths [0, n_paths_out) (test hook; each may be NULL): states_out [M][3][n_paths_out] = (x, lambda_p,
 * lambda_m) after maturity m; tangents_out [M][4][15][n_paths_out] = (dx, dlambda_p, dlambda_m, accumulated score) per direction. */
int b200sv_hawkesjd_mc_chain_greeks(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                    const double* discfactors, const int* offsets, const double* strikes, const int8_t* types, long long nb_path,
                                    int variable_type, uint64_t seed, int flags, double* prices_out, double* stderr_out, double* greeks_out,
                                    double* greeks_se_out, long long n_paths_out, double* states_out, double* tangents_out);
/* Hawkes jump-diffusion, Fourier route.  Replaces hawkesjd_chain_pricer (pricers/hawkes_jd_pricer.py:365-417) and, with a finite
 * risk_premia_gamma, hawkesjd_chain_pricer_with_risk_premia (:420-484) incl. hawkesjd_forwards_under_risk_kernel (:487-515),
 * compute_hawkes_a_mgf_grid / solve_ode_for_a (:518-641: SciPy RK45 per transform point) and the slice pricers of utils/mgf_pricer.py
 * (:174-221, :273-320).  P <= 0: 500 grid points; vol_scaler <= 0: clip(sigma, 0.2, 0.5) sqrt(min(min ttm, 1/12)) (:360-362);
 * risk_premia_gamma = NaN: no risk kernel.  a_out [M][P][3] complex128, log_mgf_out [M][P] complex128, normalizers_out / gamma_forwards_out
 * [M] are optional. */
int b200sv_hawkesjd_price_chain(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards, const double* discfactors,
                                const int* offsets, const double* strikes, const int8_t* types, int is_spot_measure, double vol_scaler, int P,
                                double risk_premia_gamma, double* prices_out, double* a_out, double* log_mgf_out, double* normalizers_out,
                                double* gamma_forwards_out);
/* prices and forward-mode sensitivities of the Hawkes Fourier chain without a risk kernel (DESIGN.md §4.3).  Arguments as in
 * b200sv_hawkesjd_price_chain; prices_out is bit-identical to it.  greeks_out [2 + 15][J], J = offsets[M]-offsets[0]: d price / d forwards[m],
 * d^2 price / d forwards[m]^2, then d price / d parameter in the order sigma, shift_p, mean_p, shift_m, mean_m, lambda_p, theta_p, kappa_p,
 * beta1_p, beta2_p, lambda_m, theta_m, kappa_m, beta1_m, beta2_m (mu does not enter the Fourier route; the compensators are differentiated
 * through shift and mean; vol_scaler and discount factors held fixed).  Optional outputs (may be NULL): dlog_mgf_out [15][M][P] complex128
 * interleaved; nfev_out [P], right-hand-side evaluations per grid point over the chain (the mesh the tangents were stepped on). */
int b200sv_hawkesjd_price_chain_greeks(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                       const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                       int is_spot_measure, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                       double* dlog_mgf_out, int* nfev_out);
/* forward-mode sensitivities of the Hawkes Fourier chain under the risk kernel exp(-gamma x) (DESIGN.md §4.12): prices_out bit-identical
 * to b200sv_hawkesjd_price_chain with the same risk_premia_gamma (spot measure, calls and puts, no discount factor, as there);
 * greeks_out [2 + 16][J]: d price / d forwards[m], d^2 price / d forwards[m]^2, then d price / d (sigma, shift_p, mean_p, shift_m, mean_m,
 * lambda_p, theta_p, kappa_p, beta1_p, beta2_p, lambda_m, theta_m, kappa_m, beta1_m, beta2_m, risk_premia_gamma), exact on the solver's
 * own meshes with the grid's imaginary parts held fixed.  Optional outputs (may be NULL): dlog_mgf_out [16][M][P] complex128 interleaved;
 * dlog_norm_out [16][M][2]: the derivatives of Re log-MGF at the normaliser points -gamma and -gamma - 1 (each solved from A = 0 over
 * the full ttms[m]); nfev_out [P].  -1: a null required pointer or a non-finite risk_premia_gamma; -5: not the spot measure, or a type
 * other than call / put; sizes, maturities and strikes as b200sv_hawkesjd_price_chain.  Every check runs before any device work. */
int b200sv_hawkesjd_price_chain_risk_premia_greeks(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                                   const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                                   int is_spot_measure, double vol_scaler, int P, double risk_premia_gamma, double* prices_out,
                                                   double* greeks_out, double* dlog_mgf_out, double* dlog_norm_out, int* nfev_out);
/* second-order sensitivities of the Hawkes Fourier chain under the risk kernel (DESIGN.md §4.13).  The arguments and outputs of
 * b200sv_hawkesjd_price_chain_risk_premia_greeks (bit-identical to it), then vanna_out [16][J]: d^2 price / d forwards[m] d parameter, and
 * hessian_out [136][J]: d^2 price / d p d q for p <= q, the upper triangle row-major in the order of greeks_out's 16 parameter rows
 * ((0,0), (0,1), .., (0,15), (1,1), ..), exact on the solver's own meshes with the grid's imaginary parts held fixed.  Optional (may be
 * NULL): d2log_mgf_out [136][M][P] complex128 interleaved; d2log_norm_out [136][M][2]: the second derivatives of Re log-MGF at the
 * normaliser points -gamma and -gamma - 1.  Return codes as b200sv_hawkesjd_price_chain_risk_premia_greeks (vanna_out and hessian_out are
 * required); every check runs before any device work. */
int b200sv_hawkesjd_price_chain_risk_premia_hessian(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                                    const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                                    int is_spot_measure, double vol_scaler, int P, double risk_premia_gamma, double* prices_out,
                                                    double* greeks_out, double* dlog_mgf_out, double* dlog_norm_out, int* nfev_out,
                                                    double* vanna_out, double* hessian_out, double* d2log_mgf_out, double* d2log_norm_out);
/* second-order sensitivities of the Hawkes Fourier chain without a risk kernel (DESIGN.md §4.5).  The arguments and outputs of
 * b200sv_hawkesjd_price_chain_greeks (bit-identical to it), then vanna_out [15][J]: d^2 price / d forwards[m] d parameter, and
 * hessian_out [120][J]: d^2 price / d p d q for p <= q, the upper triangle row-major in that parameter order ((0,0), (0,1), .., (0,14),
 * (1,1), ..).  Optional (may be NULL): d2log_mgf_out [120][M][P] complex128 interleaved, the second parameter derivatives of the log-MGF
 * grid in the same order.  Exact derivatives of the scheme on the first-order route's mesh. */
int b200sv_hawkesjd_price_chain_hessian(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                        const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                        int is_spot_measure, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                        double* dlog_mgf_out, int* nfev_out, double* vanna_out, double* hessian_out, double* d2log_mgf_out);
/* compute_hawkes_a_mgf_grid / solve_a_ode_grid (pricers/hawkes_jd_pricer.py:518-579) on caller-supplied transform grids (complex128 as interleaved
 * doubles; psi may be NULL = zeros): a_inout [P][3] holds A(0) on entry and A(dtau) on return, log_mgf_out [P] = a0 + a_p lambda_p + a_m lambda_m */
int b200sv_hawkesjd_mgf_grid(const double* phi, const double* psi, int P, double dtau, double* a_inout, const b200sv_hawkes_params* params,
                             double* log_mgf_out);
/* slice_pricer_with_mgf_grid_with_gamma (utils/mgf_pricer.py:273-320) on caller-supplied grids (complex128 as interleaved doubles) */
int b200sv_fourier_gamma(const double* log_mgf, const double* phi, int P, double risk_premia_gamma, double forward, double normalizer,
                         double gamma_forward, const double* strikes, const int8_t* types, int J, int is_spot_measure, double* prices_out);
int b200sv_hawkesjd_terminal(const b200sv_hawkes_params* params, double ttm, long long nb_path, uint64_t seed, int flags, int slice_index,
                             int use_initial_arrays, double* x_inout, double* lambda_p_inout, double* lambda_m_inout);
int b200sv_hawkesjd_step_fixed(double* x, double* lambda_p, double* lambda_m, const double* W0, const double* U_P, const double* U_M,
                               const double* J_P, const double* J_M, int S, long long N, double dt, const b200sv_hawkes_params* params);
/* Exact event-driven Monte Carlo of the Hawkes jump-diffusion (DESIGN.md §3.13): no time grid.  Per path and maturity interval the jumps
 * are simulated event by event by thinning against the sum over both intensities of the largest value of their deterministic path until
 * the interval end (max(lambda, theta, 0) for kappa >= 0, max(lambda, lambda(T), 0) for kappa < 0, any sign of kappa is exact), the
 * intensities move in closed form between events, the compensator c lambda (c = e^shift / (1 - mean) - 1) is integrated exactly and the diffusion is one
 * fp64 normal per interval.  The continuous-time limit of b200sv_hawkesjd_mc_chain's Euler step; where the intensities cannot become
 * negative (lambda0, theta >= 0, beta1_p, beta1_m >= 0, beta2_p, beta2_m <= 0) the model the Fourier route prices.  Draws: Philox keyed
 * by seed, counter (global path id, candidate index | 0xFFFFFFFF for the normal, maturity index | 0xC0000000), so results do not depend
 * on the launch shape or on sharding.  flags: fp64 state only (B200SV_STATE_F32 returns -1); the B200SV_GAUSS_* bits are not consulted.
 * max_candidates: candidates per path and maturity interval before the call fails; <= 0 selects the default 2^20.  A path that reaches
 * it stops and the call returns -6 without writing prices_out / stderr_out or the state arrays.
 * b200sv_hawkesjd_mc_chain_exact = b200sv_hawkesjd_mc_chain on the exact route (arguments as there, then the budget).  Optional test hooks
 *                              for paths [0, n_paths_out) (each may be NULL): states_out [M][3][n_paths_out] = (x, lambda_p, lambda_m) after
 *                              maturity m, events_out [M][3][n_paths_out] = (accepted '+', accepted '-', candidates) in interval m, as doubles.
 * b200sv_hawkesjd_terminal_exact = b200sv_hawkesjd_terminal on the exact route over one interval of length ttm, with the same
 *                              use_initial_arrays convention. */
int b200sv_hawkesjd_mc_chain_exact(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards, const double* discfactors,
                                   const int* offsets, const double* strikes, const int8_t* types, long long nb_path, int variable_type,
                                   uint64_t seed, int flags, double* prices_out, double* stderr_out, long long max_candidates,
                                   long long n_paths_out, double* states_out, double* events_out);
int b200sv_hawkesjd_terminal_exact(const b200sv_hawkes_params* params, double ttm, long long nb_path, uint64_t seed, int flags, int slice_index,
                                   int use_initial_arrays, long long max_candidates, double* x_inout, double* lambda_p_inout,
                                   double* lambda_m_inout);
int b200sv_hawkesjd_device_draws(uint64_t seed, long long path0, long long n, int slice, int S, double dt, const b200sv_hawkes_params* params,
                                 int flags, double* W0, double* U_P, double* U_M, double* J_P, double* J_M);

/* moments_out[2] (device) = (sum over non-NaN paths of forward*exp(x), count) for externally produced float64 states. */
int b200sv_dev_spot_moments(const double* x, long long n, double forward, double* moments_out, void* stream);

/* Sharded slices of the two neighbouring Monte Carlo routes (SURVEY.md 8e applied to 8f #4), same contract as b200sv_dev_logsv_slice:
 * local paths [0, n_local) with global ids from path_offset, float64 device state, moments_out[2] (device) = this rank's re-centring
 * moments, published to the peer-memory mailbox when p2p_ctx is given; b200sv_dev_payoff_sums / _finalize complete the maturity.
 *  - Hawkes jump-diffusion (replaces the loop body of hawkes_jd_pricer.py:687-715): state (x, lambda_p, lambda_m); init != 0 starts from
 *    (0, params->lambda_p, params->lambda_m).
 *  - rough LogSV (logsv_pricer.py:1199-1216 -> rough_logsv/split_simulation.py:466): EVERY maturity restarts at t = 0 on its own grid
 *    (nsteps steps of size h) and draws from slice 0 of the path's stream; vol_factors is [n_factors][n_local] (may be NULL),
 *    weights / nodes are HOST arrays of n_factors entries.  The payoff uses (log_spot, qvar) and, as in the reference on this route,
 *    total_paths = 1 in b200sv_dev_payoff_finalize (its "standard errors" carry no 1/sqrt(N)). */
int b200sv_dev_hawkesjd_slice(double* x, double* lambda_p, double* lambda_m, long long n_local, long long path_offset, int init,
                              const b200sv_hawkes_params* params, int nsteps, double dt, int slice_index, double forward, uint64_t seed,
                              int flags, double* moments_out, void* p2p_ctx, void* stream);
/* the device-level twin of b200sv_dev_hawkesjd_slice on the exact route (b200sv_hawkesjd_mc_chain_exact): one maturity interval of length
 * tau, max_candidates as there; overflow is a device int the kernel sets to nonzero when a path ran out of candidates (the caller zeroes
 * it before the chain and checks it after synchronising: a nonzero flag means the prices must not be used). */
int b200sv_dev_hawkesjd_exact_slice(double* x, double* lambda_p, double* lambda_m, long long n_local, long long path_offset, int init,
                                    const b200sv_hawkes_params* params, double tau, int slice_index, double forward, uint64_t seed,
                                    long long max_candidates, int* overflow, double* moments_out, void* p2p_ctx, void* stream);
int b200sv_dev_rough_logsv_slice(double* log_spot, double* vol_factors, double* qvar, long long n_local, long long path_offset,
                                 const b200sv_logsv_params* params, int n_factors, const double* weights, const double* nodes, int nsteps,
                                 double h, double forward, uint64_t seed, int flags, double* moments_out, void* p2p_ctx, void* stream);

/* test hook: out[2i] = exp(L[i]), out[2i+1] = exp(-L[i]) through the stepper's shared-polynomial exp pair (host arrays). */
int b200sv_debug_exp_pair(const double* L, long long n, double* out);
/* same for the variant the stepper runs on its table-unit state: out[2i] = exp(Ls[i] ln2/256), out[2i+1] = exp(-Ls[i] ln2/256) */
int b200sv_debug_exp_pair_scaled(const double* Ls, long long n, double* out);
/* test hook: the Box-Muller device functions on caller-chosen Philox output words (words [n][4] = r0..r3, host; z_out [n][4] host doubles).
 * flags B200SV_GAUSS_F64: box_muller_f64_fast(r0..r3) -> (z0, z1, NaN, NaN); B200SV_GAUSS_F64_PAIRED: box_muller_f64_u32 on (r0, r1) and on
 * (r2, r3); otherwise the default float draw box_muller_f32 on the same two pairs.  The shared tables are initialised as in the kernels. */
int b200sv_debug_box_muller(const uint32_t* words, long long n, int flags, double* z_out);
/* test hook: out[i] = op(a[i], b[i]) through the fp64 device helpers (host arrays; b is read by B200SV_DEBUG_FAST_DIV only, else may be NULL):
 * fast_div(a, b), fast_sqrt(a), fast_sqrt_pos(a), neg2_log(a) = -2 ln(a), exp_table(a) */
enum { B200SV_DEBUG_FAST_DIV = 0, B200SV_DEBUG_FAST_SQRT = 1, B200SV_DEBUG_FAST_SQRT_POS = 2, B200SV_DEBUG_NEG2_LOG = 3, B200SV_DEBUG_EXP_TABLE = 4 };
int b200sv_debug_fastmath(int op, const double* a, const double* b, long long n, double* out);
/* test hook: the Hawkes stepper's jump-clock functions on caller-chosen 32-bit words r[i] against intensities lambda[i] at step dt (host
 * arrays; params supplies shift / mean of the sizes).  out[n][6] = u = (r + 1/2) 2^-32, the clock -ln(u)/dt, the jump sizes
 * shift_p + mean_p (-ln u) and shift_m - (-mean_m)(-ln u) as b200sv_hawkesjd_device_draws exports them, then 1.0 / 0.0 for the candidate
 * filter on the raw word and for the fused firing decision of the in-kernel stepper, which must equal lambda > clock. */
int b200sv_debug_hawkes_clocks(const uint32_t* r, const double* lambda, long long n, double dt, const b200sv_hawkes_params* params, double* out);

/* ------------------------------------------------------------------------------------------------------------------
 * Fourier / MGF, host-level
 * ------------------------------------------------------------------------------------------------------------------ */

/* replaces logsv_chain_pricer (pricers/logsv_pricer.py:669-739), LOG_RETURN and Q_VAR branches: transform grid
 * (utils/mgf_pricer.py:11-34), per maturity the affine-expansion ODEs integrated with SciPy's RK45 control law
 * (pricers/logsv/affine_expansion.py:229-303, 492-529) carried across maturities, log-MGF contraction (:674-685)
 * and the Simpson/Fourier sums (utils/mgf_pricer.py:174-221).  vol_scaler <= 0 selects set_vol_scaler (:664-666).
 * variable_type = B200SV_Q_VAR prices calls on the annualised quadratic variance on the psi grid -0.5 + 1j*linspace(0, 4000, P)
 * (utils/mgf_pricer.py:37-47, :323-358; only 'C' payoffs, else -5) with phi = 0 (MMA) / 1 (inverse measure) (:79-85).
 * P = grid size, <= 0 selects the reference's (1000 for LOG_RETURN, 40000 for Q_VAR).  Optional outputs (may be NULL):
 * a_out [M][P][n] complex128 interleaved, log_mgf_out [M][P] complex128 interleaved. */
int b200sv_logsv_price_chain(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                             const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                             const int8_t* types, int is_spot_measure, int variable_type, int expansion_order,
                             double vol_scaler, int P, double* prices_out, double* a_out, double* log_mgf_out);

/* replaces heston_chain_pricer, LOG_RETURN and Q_VAR branches (pricers/heston_pricer.py:217-282) with compute_heston_mgf_grid
 * (:183-214).  vol_scaler <= 0 selects min(0.3, sqrt(v0*ttms[0])) (:234-235). */
int b200sv_heston_price_chain(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                              const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                              int variable_type, double vol_scaler, int P, double* prices_out, double* log_mgf_out);

/* prices and forward-mode sensitivities of the two Fourier chain pricers above (DESIGN.md §4.2), LOG_RETURN only (else -4).  Arguments as
 * in b200sv_*_price_chain; prices_out is bit-identical to it.  greeks_out [2 + n][J], J = offsets[M]-offsets[0]: d price / d forwards[m],
 * d^2 price / d forwards[m]^2, then d price / d parameter in struct field order (n = 6 LogSV, 5 Heston; vol_scaler, etas and discount
 * factors held fixed).  Optional outputs (may be NULL): dlog_mgf_out [n][M][P] complex128 interleaved, the parameter derivatives of the
 * log-MGF grid; nfev_out [P], right-hand-side evaluations per grid point over the chain (the mesh the tangents were stepped on). */
int b200sv_logsv_price_chain_greeks(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                    const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                    const int8_t* types, int is_spot_measure, int variable_type, int expansion_order,
                                    double vol_scaler, int P, double* prices_out, double* greeks_out, double* dlog_mgf_out,
                                    int* nfev_out);
int b200sv_heston_price_chain_greeks(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                     const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                     int variable_type, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                     double* dlog_mgf_out);

/* second-order forward-mode sensitivities of the two Fourier chain pricers (DESIGN.md §4.4), LOG_RETURN only (else -4).  The arguments
 * and outputs of b200sv_*_price_chain_greeks (bit-identical to it), then vanna_out [n][J]: d^2 price / d forwards[m] d parameter, and
 * hessian_out [n(n+1)/2][J]: d^2 price / d p d q for p <= q, the upper triangle row-major in struct field order ((0,0), (0,1), ..,
 * (0,n-1), (1,1), ..).  Optional (may be NULL): d2log_mgf_out [n(n+1)/2][M][P] complex128 interleaved, the second parameter
 * derivatives of the log-MGF grid in the same order.  Exact derivatives of the scheme on the first-order route's mesh. */
int b200sv_logsv_price_chain_hessian(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                     const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                     const int8_t* types, int is_spot_measure, int variable_type, int expansion_order,
                                     double vol_scaler, int P, double* prices_out, double* greeks_out, double* dlog_mgf_out,
                                     int* nfev_out, double* vanna_out, double* hessian_out, double* d2log_mgf_out);
int b200sv_heston_price_chain_hessian(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                      const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                      int variable_type, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                      double* dlog_mgf_out, double* vanna_out, double* hessian_out, double* d2log_mgf_out);

/* theta of the Fourier chain pricers (DESIGN.md §4.8), LOG_RETURN only (else -4).  The arguments and outputs of the _greeks twin
 * (bit-identical to it), then theta_out [J]: -d price / d ttms[m] per year, with the slice forward and discount factor, the earlier
 * maturities, etas and the transform grid held (vol_scaler <= 0 resolved on the unmoved chain); the adaptive routes hold the accepted mesh
 * of slice m and move its last step only.  Optional (may be NULL): dlog_mgf_theta_out [M][P] complex128 interleaved, d log_mgf / d ttms[m]
 * of slice m; theta_nfev_out [P] (LogSV, Hawkes), the right-hand-side evaluations of the theta kernel's own primal solve per grid point,
 * equal to nfev_out when it ran the pricing mesh. */
int b200sv_logsv_price_chain_greeks_theta(const b200sv_logsv_params* params, int M, const double* ttms, const double* forwards,
                                          const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                          const int8_t* types, int is_spot_measure, int variable_type, int expansion_order,
                                          double vol_scaler, int P, double* prices_out, double* greeks_out, double* dlog_mgf_out,
                                          int* nfev_out, double* theta_out, double* dlog_mgf_theta_out, int* theta_nfev_out);
int b200sv_heston_price_chain_greeks_theta(const b200sv_heston_params* params, int M, const double* ttms, const double* forwards,
                                           const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                           int variable_type, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                           double* dlog_mgf_out, double* theta_out, double* dlog_mgf_theta_out);
int b200sv_hawkesjd_price_chain_greeks_theta(const b200sv_hawkes_params* params, int M, const double* ttms, const double* forwards,
                                             const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                             int is_spot_measure, double vol_scaler, int P, double* prices_out, double* greeks_out,
                                             double* dlog_mgf_out, int* nfev_out, double* theta_out, double* dlog_mgf_theta_out,
                                             int* theta_nfev_out);

/* B parameter sets on ONE chain in one pass -- the objective of the calibration drivers and its finite-difference gradient:
 * _LogSvCalibrationObjective.__call__ (pricers/logsv_pricer.py:234-294: compute_model_ivols_for_chain = logsv_chain_pricer +
 * option_chain.compute_model_ivols_from_chain_data), which scipy SLSQP evaluates n+1 times per iteration, one parameter set at a time.
 * params[B]; etas[B*M] (NULL = 1); prices_out[B*J], ivols_out[B*J] (NULL = skip the fused Black-76 inversion), J = offsets[M]-offsets[0],
 * row b in chain order.  vol_scaler <= 0: each set gets its own default grid sigma0_b*sqrt(min(min ttm, 1/24)) (:664-666).
 * LOG_RETURN only.  Row b equals b200sv_logsv_price_chain(params[b]) (+ b200sv_bsm_implied_vols) bit for bit. */
int b200sv_logsv_price_chain_batch(const b200sv_logsv_params* params, int B, int M, const double* ttms, const double* forwards,
                                   const double* discfactors, const double* etas, const int* offsets, const double* strikes,
                                   const int8_t* types, int is_spot_measure, int expansion_order, double vol_scaler, int P,
                                   double* prices_out, double* ivols_out);

/* same for Heston: the objective of HestonPricer.calibrate_model_params_to_chain (pricers/heston_pricer.py:111-180). */
int b200sv_heston_price_chain_batch(const b200sv_heston_params* params, int B, int M, const double* ttms, const double* forwards,
                                    const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                    double vol_scaler, int P, double* prices_out, double* ivols_out);

/* B parameter sets over K chains in one call -- the objectives of K calibrations run in lock-step, one call per optimizer round.  Set b
 * is priced on chain chain_of_set[b] (0 <= . < K).  The chains are concatenated: chain k has Ms[k] maturities at ttms / forwards /
 * discfactors [Ms[0] + .. + Ms[k-1]] and its Ms[k] + 1 offsets into strikes / types at offsets [(Ms[0] + 1) + .. + (Ms[k-1] + 1)].  Every
 * Ms[k] must be >= 1, since it places the chains after k; of a chain that no set points at nothing else is read.  LogSV etas (NULL = 1):
 * each set's own Ms[chain_of_set[b]] backbone values, set after set.
 * vol_scalers[K]: the grid of each chain's sets, <= 0 for each set's own default grid.  prices_out / ivols_out (NULL = skip the fused
 * Black-76 inversion): the rows of the sets one after the other, set b's row holding the J of its own chain.  LOG_RETURN only.
 * Row b equals, bit for bit, row i of b200sv_*_price_chain_batch called on chain chain_of_set[b] with the sets of this call on that chain,
 * in call order, b being the i-th of them: whatever else shares the call. */
int b200sv_logsv_price_chains_batch(const b200sv_logsv_params* params, int B, const int* chain_of_set, int K, const int* Ms,
                                    const double* ttms, const double* forwards, const double* discfactors, const double* etas,
                                    const int* offsets, const double* strikes, const int8_t* types, int is_spot_measure, int expansion_order,
                                    const double* vol_scalers, int P, double* prices_out, double* ivols_out);
int b200sv_heston_price_chains_batch(const b200sv_heston_params* params, int B, const int* chain_of_set, int K, const int* Ms,
                                     const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                     const double* strikes, const int8_t* types, const double* vol_scalers, int P, double* prices_out,
                                     double* ivols_out);
/* the Hawkes twin, without a risk kernel: layout, vol_scalers and row equality as above, against b200sv_hawkesjd_price_chain_batch with
 * gammas = NULL (P <= 0: 500).  Each chain's sets are integrated by one Riccati launch. */
int b200sv_hawkesjd_price_chains_batch(const b200sv_hawkes_params* params, int B, const int* chain_of_set, int K, const int* Ms,
                                       const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                       const double* strikes, const int8_t* types, int is_spot_measure, const double* vol_scalers, int P,
                                       double* prices_out, double* ivols_out);
/* ... and under the risk kernel: gammas [B] (all finite) the risk_premia_gamma of each set, spot measure and 'C' / 'P' only (else -5), row
 * equality against b200sv_hawkesjd_price_chain_batch with gammas.  One Riccati launch per chain plus two: every (set, maturity)
 * normaliser solve of the call in one launch, and one Fourier-sum launch. */
int b200sv_hawkesjd_price_chains_batch_gamma(const b200sv_hawkes_params* params, const double* gammas, int B, const int* chain_of_set, int K,
                                             const int* Ms, const double* ttms, const double* forwards, const double* discfactors,
                                             const int* offsets, const double* strikes, const int8_t* types, int is_spot_measure,
                                             const double* vol_scalers, int P, double* prices_out, double* ivols_out);

/* same for the Hawkes jump-diffusion: the objectives of HawkesJDPricer.calibrate_model_params_to_chain and
 * calibrate_risk_premia_gamma_to_chain (pricers/hawkes_jd_pricer.py:230-357).  B Hawkes parameter sets on one chain in one pass.
 * gammas: NULL = no risk kernel, else [B] finite risk_premia_gamma per set (all sets on the risk-kernel route: 'C' / 'P' under the spot
 * measure only, else -5).  vol_scaler <= 0: per-set default grid clip(sigma_b, 0.2, 0.5) sqrt(min(min ttm, 1/12)); with gammas every set
 * has its own grid (Re phi = -1/2 - gamma_b) either way.  P <= 0: 500 grid points.  prices_out [B][J], ivols_out [B][J] (NULL = skip the
 * fused Black-76 inversion), row b in chain order.  Row b equals b200sv_hawkesjd_price_chain(params[b], gammas ? gammas[b] : NaN)
 * (+ b200sv_bsm_implied_vols on the chain's forwards / discfactors) bit for bit. */
int b200sv_hawkesjd_price_chain_batch(const b200sv_hawkes_params* params, int B, int M, const double* ttms, const double* forwards,
                                      const double* discfactors, const int* offsets, const double* strikes, const int8_t* types,
                                      int is_spot_measure, double vol_scaler, int P, const double* gammas,
                                      double* prices_out, double* ivols_out);

/* replaces compute_logsv_a_mgf_grid, non-analytic branch (pricers/logsv/affine_expansion.py:570-685 -> solve_a_ode_grid
 * :492-529): phi, psi, a (in: A(0), out: A(dtau)), log_mgf_out are complex128 interleaved host arrays of P, P, P*n, P. */
int b200sv_logsv_mgf_grid(const double* phi, const double* psi, int P, double dtau, double* a_inout,
                          const b200sv_logsv_params* params, double eta, int is_spot_measure, int expansion_order,
                          double* log_mgf_out);

/* compute_logsv_a_mgf_grid(is_analytic=True): the semi-analytic branch solve_analytic_ode_for_a (pricers/logsv/affine_expansion.py:306-384) over a
 * transform grid -- business-day steps (year_days = 260 in the reference), linear part exact, quadratic part by 10 fixed-point sweeps.
 * a_inout complex [P][n] in/out, log_mgf_out complex [P]; vol_backbone_eta is ignored on this branch, as in the reference. */
int b200sv_logsv_mgf_grid_analytic(const double* phi, const double* psi, int P, double dtau, double* a_inout, const b200sv_logsv_params* params,
                                   int is_spot_measure, int expansion_order, int year_days, double* log_mgf_out);
/* compute_logsv_a_mgf_grid(is_stiff_solver=True): solve_ivp(method="BDF", jac=func_rhs_jac) per grid point (pricers/logsv/affine_expansion.py:229-303) --
 * a clone of SciPy's BDF control law (scipy 1.18.1 _ivp/bdf.py), default rtol 1e-3 / atol 1e-6.  Same arrays as b200sv_logsv_mgf_grid. */
int b200sv_logsv_mgf_grid_bdf(const double* phi, const double* psi, int P, double dtau, double* a_inout, const b200sv_logsv_params* params,
                              double eta, int is_spot_measure, int expansion_order, double* log_mgf_out);
/* func_a_ode_quadratic_terms (pricers/logsv/affine_expansion.py:67-184): the dense coefficient tensors of A' = A^T M^(k) A + L A + H for
 * P transform points, n = 3 (FIRST) or 5 (SECOND): M_out complex [P][n][n][n] (symmetric in the last two indices), L_out [P][n][n],
 * H_out [P][n], interleaved (re, im).  psi may be NULL (zeros).  Parity entry: the pricing kernels integrate the same rows in sparse form. */
int b200sv_logsv_ode_terms(const double* phi, const double* psi, int P, const b200sv_logsv_params* params, double eta, int is_spot_measure,
                           int expansion_order, double* M_out, double* L_out, double* H_out);
/* func_rhs (affine_expansion.py:187-205) evaluated by the production right-hand side at A [P][n] complex -> rhs_out [P][n] complex. */
int b200sv_logsv_ode_rhs(const double* phi, const double* psi, int P, const double* A, const b200sv_logsv_params* params, double eta,
                         int is_spot_measure, int expansion_order, double* rhs_out);
/* func_rhs with the reference's own signature (caller-supplied dense complex tensors M [n][n][n], L [n][n], H [n]; A [P][n]) */
int b200sv_ode_rhs_dense(const double* A, int P, int n, const double* M, const double* L, const double* H, double* rhs_out);

/* replaces compute_heston_mgf_grid (pricers/heston_pricer.py:183-214); a, b in/out complex128[P]. */
int b200sv_heston_mgf_grid(const double* phi, const double* psi, int P, double dtau, double* a_inout, double* b_inout,
                           const b200sv_heston_params* params, double* log_mgf_out);

/* replaces vanilla_slice_pricer_with_mgf_grid (utils/mgf_pricer.py:174-221). */
int b200sv_fourier_vanilla(const double* log_mgf, const double* phi, int P, double forward, const double* strikes,
                           const int8_t* types, int J, double discfactor, int is_spot_measure, double* prices_out);

/* replaces slice_qvar_pricer_with_a_grid (utils/mgf_pricer.py:323-358): calls on annualised quadratic variance from the log-MGF on
 * the psi grid; price = max(discfactor * S / ttm, 1e-10), S = nansum Re((dp/pi)/psi^2 * exp(K*ttm*psi + log_mgf)). */
int b200sv_fourier_qvar(const double* log_mgf, const double* psi, int P, double ttm, const double* strikes,
                        const int8_t* types, int J, double discfactor, double* prices_out);

/* the sum of pdf_with_mgf_grid (utils/mgf_pricer.py:361-384): out[j] = nansum Re((dp/pi) * exp(z[j]*grid + log_mgf)); the caller
 * applies z = (x - shift)/scale beforehand and the dx / scale factors afterwards (pricers/logsv_pricer.py:778-803). */
int b200sv_fourier_pdf(const double* log_mgf, const double* grid, int P, const double* z, int J, double* out);

/* replaces digital_slice_pricer_with_mgf_grid (utils/mgf_pricer.py:224-269). */
int b200sv_fourier_digital(const double* log_mgf, const double* phi, int P, double forward, const double* strikes,
                           const int8_t* types, int J, double discfactor, double* prices_out);

/* ------------------------------------------------------------------------------------------------------------------
 * Black-76 implied volatilities (the step after every chain pricer in the reference's callers)
 * ------------------------------------------------------------------------------------------------------------------ */

/* replaces option_chain.compute_model_ivols_from_chain_data (data/option_chain.py:327-346 -> third-party
 * vanilla_option_pricers.infer_bsm_ivols_from_model_chain_prices): prices[] and ivols_out[] are flat in chain order
 * (offsets[M]-offsets[0] entries).  'IC'/'IP' quotes are inverted like 'C'/'P'; prices outside the no-arbitrage bounds give NaN. */
int b200sv_bsm_implied_vols(int M, const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                            const double* strikes, const int8_t* types, const double* prices, double* ivols_out);
/* test hook: b200sv_bsm_implied_vols plus iterations_out[] = the Newton iterations each quote took (0 for a NaN verdict) */
int b200sv_debug_bsm_implied_vols(int M, const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                  const double* strikes, const int8_t* types, const double* prices, double* ivols_out, int* iterations_out);
/* implied-vol sensitivities of model prices, for any model (DESIGN.md §4.6).  The chain and prices[] as b200sv_bsm_implied_vols; NP
 * (1..15, else -1) model parameters; greeks [2+NP][J] = d price / d forwards[m], d^2 price / d forwards[m]^2, d price / d p, in exactly the
 * layout b200sv_*_price_chain_greeks return; optional vanna [NP][J] and hessian [NP(NP+1)/2][J] (upper triangle, row-major) in the layout of
 * b200sv_*_price_chain_hessian, given together or not at all (else -1), each with its output (else -1).  Outputs: ivols_out [J], bit-identical
 * to b200sv_bsm_implied_vols on the same prices; ivol_greeks_out [2+NP][J], ivol_vanna_out [NP][J], ivol_hessian_out [NP(NP+1)/2][J]: the
 * same derivatives of the implied vol (sticky strike: the forward moves the model price and Black's forward).  A NaN ivol gives NaN rows; an
 * ivol at an end of the inversion bracket (1e-8 or 10) gives zero rows.  Unknown type codes: -3. */
int b200sv_bsm_implied_vol_sensitivities(int M, const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                         const double* strikes, const int8_t* types, const double* prices, int NP, const double* greeks,
                                         const double* vanna, const double* hessian, double* ivols_out, double* ivol_greeks_out,
                                         double* ivol_vanna_out, double* ivol_hessian_out);
/* implied-vol theta (DESIGN.md §4.8).  The chain and prices[] as b200sv_bsm_implied_vols, theta [J] = -d price / d ttms[m] as the
 * b200sv_*_price_chain_greeks_theta entry points return it.  Outputs: ivols_out [J], bit-identical to b200sv_bsm_implied_vols, and
 * ivol_theta_out [J] = -d ivol / d ttms[m] = (theta + d B / d ttm) / vega, B the discounted Black-76 price at the same discount factor.  NaN
 * where the ivol is NaN, 0 where it is an end of the inversion bracket (1e-8 or 10).  Unknown type codes: -3. */
int b200sv_bsm_implied_vol_theta(int M, const double* ttms, const double* forwards, const double* discfactors, const int* offsets,
                                 const double* strikes, const int8_t* types, const double* prices, const double* theta, double* ivols_out,
                                 double* ivol_theta_out);

#ifdef __cplusplus
}
#endif
#endif /* B200SV_H */
