// NRMP kernel: one warp solves one environment's convex program per launch.
//
// Replaces NRMP.forward (neupan/blocks/nrmp.py:114-150) including
//   robot.generate_state_parameter_value / linear_{ackermann,diff,omni}_model  robot.py:239-316
//   NRMP.generate_coefficient_parameter_value (fa, fb, padding)                nrmp.py:220-261
//   the cvxpylayers -> diffcp -> ECOS solve of the program built at           nrmp.py:263-383,
//                                                                              robot.py:73-236
//   PAN.stop_criteria                                                          pan.py:215-243
//
// Method: the states are eliminated through the linearised dynamics, s_{t+1} = s0_{t+1} + F_t u.  The squared
// hinge of robot.py:183-198,  (rho/2) max(0, r)^2 with r_tm = D_t + fb_tm - fa_tm.s_{t+1,xy},  is written as
// min_w (rho/2) w^2 s.t. w >= r  -- ONE inequality per hinge (w >= 0 is redundant: for r <= 0 the unconstrained
// minimiser w = 0 is feasible) -- and w is eliminated through its stationarity condition w = z/rho, z the row's
// multiplier, so a hinge row carries only the pair (s, z) with  s = z/rho - r >= 0.  [The CPU checker oracle/ipm.py
// keeps the textbook two-row lift (w >= 0, w >= r): every inactive hinge is then a degenerate pair (s_w, z_w -> 0
// together like sqrt(mu)) and the interior point iteration converges linearly, ~16.5 iterations on C4; the one-row
// form is non-degenerate, converges superlinearly at the end (~14 cold) and has half the hinge state.  The two
// formulations are independent derivations of the same program -- their agreement is a parity check, not shared
// algebra.]  A Mehrotra predictor-corrector primal-dual interior point method runs in FP64 from a strictly feasible
// start: cold (u = 0, D mid-range) or WARM from the previous PAN iteration's solution of the same environment
// (x pulled 5 % towards the centre, slacks recomputed from it, multipliers floored at mu0 / s): ~10 iterations.
// Inside each Newton step the T*M hinge rows and the T distances D_t are eliminated analytically (both blocks are
// diagonal), so the only factorisation is a dense 2T x 2T Cholesky: blocked, in the registers of the tensor-pipe assembly, for
// the compile-time (T, M) specialisations; in the warp's shared memory otherwise.
//
// Mapping: lanes own rows of the 2T x 2T system (triangular solves run in registers with
// shuffles), lanes own HPL hinge rows each whose slack/multiplier state lives in registers, lanes
// own horizon steps for the per-step reductions.  Inverse slacks and step ratios are float (they only
// shape the Newton direction / step length; residuals and iterates are FP64), reciprocals use
// rcp.approx + Newton.  All synchronisation is __syncwarp; a warp finishes independently.
#pragma once
#include "nrmp_common.cuh"

namespace nb {

#define NB_LL(i, n) _Pragma("unroll 1") for (int i = lane; i < (n); i += 32)
// the lane loop of the interior point iteration: with compile-time shapes (kFixed, nrmp_solve_env) it has a fixed trip count, is
// unrolled, and each step is predicated on the lane's row existing; otherwise it is NB_LL
#define NB_LW(i, n)                                                                 \
  _Pragma("unroll(kLaneUnroll)") for (int i##_b = kFixed ? 0 : lane; i##_b < (n); i##_b += 32) \
    if (const int i = i##_b + (kFixed ? lane : 0); i < (n))

// NB_NRMP_PHASES (timing only, off by default): each warp adds the clock64() cycles it spends in the setup (sections 1-5) and in
// the phases (a)-(e) of the interior point iteration to nb_nrmp_phase_cycles[0..5], [6] counts the iterations that ran (e) and
// [7] the setups.  Read back through nb_nrmp_read_phases (nrmp.cu); tools/nrmp_bench.py --phases builds and reads that variant.
// The arithmetic is untouched, so results are the same with the flag on.
#ifndef NB_NRMP_PHASES
#define NB_NRMP_PHASES 0
#endif
#if NB_NRMP_PHASES
__device__ unsigned long long nb_nrmp_phase_cycles[8];
#define NB_PHASE(p)                                                                                    \
  do {                                                                                                 \
    const long long now_ = clock64();                                                                  \
    if (lane == 0) atomicAdd(&nb_nrmp_phase_cycles[p], (unsigned long long)(now_ - phase_t0));         \
    if (lane == 0 && ((p) == 0 || (p) == 5)) atomicAdd(&nb_nrmp_phase_cycles[(p) == 0 ? 7 : 6], 1ull); \
    phase_t0 = clock64();                                                                              \
  } while (0)
#else
#define NB_PHASE(p) \
  do {              \
  } while (0)
#endif

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_maxf(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// 1/x for a normal positive double: hardware seed (~20 bits) + two Newton steps
__device__ __forceinline__ double rcp64(double x) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  r = fma(fma(-x, r, 1.0), r, r);
  r = fma(fma(-x, r, 1.0), r, r);
  return r;
}
// 1/sqrt(x) for a positive double inside float range: float seed (2 ulp, ~22 bits) + two Newton steps (44, then > 53 bits)
__device__ __forceinline__ double rsqrt64(double x) {
  double r = (double)rsqrtf((float)x);
  const double hx = -0.5 * x;
#pragma unroll
  for (int i = 0; i < 2; ++i) r = r * fma(hx, r * r, 1.5);
  return r;
}
// D (8x8, FP64) += A (8x4, row) * B (4x8, col) on the FP64 tensor pipe.  Lane l = 4 g + q holds A[g][q], B[q][g], D[g][2q], D[g][2q+1].
__device__ __forceinline__ void dmma884(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
__device__ __forceinline__ float rcpf(double x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"((float)x));
  return r;
}

// ---- stop criterion of one environment (pan.py:215-243) and the update of PAN.current_nom_values: one warp.  Called at the end of the
// solve, or -- NrmpParams::defer_stop -- from nrmp_stop_kernel: the ~1300 floats it reads per environment are latency the solve
// kernel cannot hide (6.8 % of its warp time on C4), a bandwidth kernel over the batch reads them in a few microseconds.
template <int TT, int MM>
__device__ __forceinline__ void nrmp_stop_env(const NrmpParams& prm, const int b, const int lane) {
  const int T = TT > 0 ? TT : prm.T, M = TT > 0 ? MM : prm.M, T1 = T + 1;
  const float* os = prm.out_s + (size_t)b * 3 * T1;
  const float* ou = prm.out_u + (size_t)b * 2 * T;
  if (prm.prev_valid) {
    const int E = prm.E;
    const int cur_cnt = (prm.fa || M == 0 || !prm.sel_count) ? 0 : prm.sel_count[b];
    const int valid = prm.prev_valid[b];
    const int pcnt = prm.prev_count[b];
    float* ps = prm.prev_s + (size_t)b * 3 * T1;
    float* pu_ = prm.prev_u + (size_t)b * 2 * T;
    float* pmu = prm.prev_mu ? prm.prev_mu + (size_t)b * T1 * M * E : nullptr;
    float* plam = prm.prev_lam ? prm.prev_lam + (size_t)b * T1 * M * 2 : nullptr;
    const float* cmu = prm.sel_mu ? prm.sel_mu + (size_t)b * T1 * M * E : nullptr;
    const float* clam = prm.sel_lam ? prm.sel_lam + (size_t)b * T1 * M * 2 : nullptr;
    float diff = 0.f;
    if (valid) {
      if (cur_cnt == 0 || pcnt == 0) {
        double a1 = 0, a2 = 0;
        NB_LL(i, 3 * T1) { const double d = (double)os[i] - (double)ps[i]; a1 += d * d; }
        NB_LL(i, 2 * T) { const double d = (double)ou[i] - (double)pu_[i]; a2 += d * d; }
        const float n1f = sqrtf((float)warp_sum(a1)), n2f = sqrtf((float)warp_sum(a2));
        diff = n1f * n1f + n2f * n2f;
      } else {
        const int en = cur_cnt < pcnt ? cur_cnt : pcnt;
        double a1 = 0, a2 = 0;
        NB_LL(i, T1 * en * E) {
          const int tt = i / (en * E), rem = i - tt * en * E;  // rem = col*E + e, col < en
          const size_t o = (size_t)tt * M * E + rem;
          const double d = (double)cmu[o] - (double)pmu[o];
          a1 += d * d;
        }
        NB_LL(i, T1 * en * 2) {
          const int tt = i / (en * 2), rem = i - tt * en * 2;
          const size_t o = (size_t)tt * M * 2 + rem;
          const double d = (double)clam[o] - (double)plam[o];
          a2 += d * d;
        }
        const float md = sqrtf((float)warp_sum(a1)) / (float)en, ld = sqrtf((float)warp_sum(a2)) / (float)en;
        diff = md * md + ld * ld;
      }
    }
    __syncwarp();
    NB_LL(i, 3 * T1) ps[i] = os[i];
    NB_LL(i, 2 * T) pu_[i] = ou[i];
    if (pmu && cmu) {
      NB_LL(i, T1 * M * E) pmu[i] = cmu[i];
      NB_LL(i, T1 * M * 2) plam[i] = clam[i];
    }
    if (lane == 0) {
      prm.prev_valid[b] = 1;
      prm.prev_count[b] = cur_cnt;
      if (valid && diff < prm.iter_threshold && prm.active) prm.active[b] = 0;
    }
  }
}

// Cholesky factor of the reduced Hessian held as the lower-triangular 8x8 tiles of the DMMA accumulators: tile (I, J), J <= I,
// at w0/w1[I(I+1)/2 + J], lane 4g + q holding rows 8I + g, columns 8J + 2q (w0) and 8J + 2q + 1 (w1).  Rows nU..8NT-1 are
// identity padding.  Right-looking by block columns: the diagonal tile and the panel below it column by column with quad
// shuffles, then the trailing SYRK / GEMM updates on the FP64 tensor pipe, L_IJ -= L_IK L_JK' as two m8n8k4 k-steps.  Their
// k-index runs over the columns in the order (2q | 2q + 1), which is the accumulator layout itself: the finished tiles are the
// operands as they are.  L goes to the staircase H[hrow(i) + j] and 1/L_ii to `invd` of lane i, as the unblocked factorisation
// leaves them.  Returns false at a pivot that is not positive (or NaN); the padding never reaches a pivot.
template <int NT, int NU>
__device__ __forceinline__ bool nrmp_block_cholesky(double (&w0)[NT * (NT + 1) / 2], double (&w1)[NT * (NT + 1) / 2], double* H, double& invd,
                                                    const int lane) {
  const int q = lane & 3, g = lane >> 2, quad = lane & ~3;
#pragma unroll
  for (int K = 0; K < NT; ++K) {
    const int kd = K * (K + 1) / 2 + K;
    const int ncol = NU - 8 * K < 8 ? NU - 8 * K : 8;  // padded columns of the last block are not factored
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (k >= ncol) break;
      const int src = k >> 1;
      const bool hi = (k & 1) != 0;
      const double piv = __shfl_sync(0xffffffffu, hi ? w1[kd] : w0[kd], 4 * k + src);
      const double c0 = __shfl_sync(0xffffffffu, hi ? w1[kd] : w0[kd], 8 * q + src);      // A_KK[2q][k]
      const double c1 = __shfl_sync(0xffffffffu, hi ? w1[kd] : w0[kd], 8 * q + 4 + src);  // A_KK[2q + 1][k]
      double own[NT];  // A_XK[g][k] of this lane's row in every tile of the block column
#pragma unroll
      for (int X = K; X < NT; ++X) {
        const int xi = X * (X + 1) / 2 + K;
        own[X] = __shfl_sync(0xffffffffu, hi ? w1[xi] : w0[xi], quad + src);
      }
      if (!(piv > 0.0)) return false;
      const double ild = rsqrt64(piv);
      if (lane == 8 * K + k) invd = ild;
      const double l0 = c0 * ild, l1 = c1 * ild;  // L_KK[2q][k], L_KK[2q + 1][k]
#pragma unroll
      for (int X = K; X < NT; ++X) {
        const int xi = X * (X + 1) / 2 + K;
        const double l = own[X] * ild;  // L_XK[g][k]
        if (q == src) {
          if (hi) w1[xi] = l; else w0[xi] = l;
        }
        if (2 * q > k) w0[xi] = fma(-l, l0, w0[xi]);
        if (2 * q + 1 > k) w1[xi] = fma(-l, l1, w1[xi]);
      }
    }
#pragma unroll
    for (int X = K; X < NT; ++X) {  // block column K is final
      const int xi = X * (X + 1) / 2 + K, i = 8 * X + g, j = 8 * K + 2 * q;
      if (i < NU && j <= i) H[((i * (i + 3)) >> 1) + j] = w0[xi];
      if (i < NU && j + 1 <= i) H[((i * (i + 3)) >> 1) + j + 1] = w1[xi];
    }
#pragma unroll
    for (int I = K + 1; I < NT; ++I) {
      const int ik = I * (I + 1) / 2 + K;
#pragma unroll
      for (int J = K + 1; J <= I; ++J) {
        const int ij = I * (I + 1) / 2 + J, jk = J * (J + 1) / 2 + K;
        dmma884(w0[ij], w1[ij], -w0[ik], w0[jk]);
        dmma884(w0[ij], w1[ij], -w1[ik], w1[jk]);
      }
    }
  }
  __syncwarp();
  return true;
}

// SMALL: 2T <= 32, every lane owns at most one row of the reduced system (one register slot in the
// triangular solves); the general version (T <= 32) carries a second slot.
// TT, MM: compile-time horizon / hinge rows per step (0 = read them from the parameters).  With constants every
// workspace offset, loop bound and row stride folds into immediates -- half of the generic kernel's
// instructions were integer address arithmetic.
// Residency: the (10, 10) specialisation is built for 5 CTAs of 3 warps (15 warps) per SM (NB_NRMP_WPC) -- 128 registers with
// ~220 B of spill stores, and ~43 KB of shared memory per CTA, which also caps the SM at 15 warps.  At B = 4096 that is 1980
// resident solves on 132 SMs.  (__maxnreg__(144) instead of the min-blocks bound makes ptxas spill more.)
template <int HPL, bool SMALL, int TT, int MM>
__device__ __forceinline__ void nrmp_solve_env(const NrmpParams& prm, const int b, double* wsp, const unsigned short* __restrict__ ptab, const int lane) {
  const int T = TT > 0 ? TT : prm.T, M = TT > 0 ? MM : prm.M, T1 = T + 1;
  const int nU = 2 * T, nR = nU - 2, TD = M > 0 ? T : 0, TM = T * M;
  const int nP = nU * (nU + 1) / 2;
  const int oBU = 0, oBL = nU, oRU = 2 * nU, oRL = oRU + nR, oDU = oRL + nR, oDL = oDU + TD;
  const int mb = oDL + TD;
  auto hrow = [](int i) { return (i * (i + 3)) >> 1; };  // offset of row i of the lower-triangular H / L
#if NB_NRMP_PHASES
  long long phase_t0 = clock64();
#endif
#ifndef NB_NRMP_DMMA
#define NB_NRMP_DMMA 1
#endif
#ifndef NB_NRMP_UNROLL_CHOL
#define NB_NRMP_UNROLL_CHOL 0
#endif
#ifndef NB_NRMP_UNROLL_SOLVE
#define NB_NRMP_UNROLL_SOLVE 1
#endif
#ifndef NB_NRMP_CHOL_TWICE
#define NB_NRMP_CHOL_TWICE 0
#endif
#ifndef NB_NRMP_BLOCKCHOL
#define NB_NRMP_BLOCKCHOL 1
#endif
  constexpr int kUnrollSolve = (TT > 0 && NB_NRMP_UNROLL_SOLVE) ? 32 : 2;
  constexpr int kUnrollCholK = (TT > 0 && NB_NRMP_UNROLL_CHOL) ? 16 : 1, kUnrollCholP = (TT > 0 && NB_NRMP_UNROLL_CHOL) ? 32 : 4;
  const bool kDmma = NB_NRMP_DMMA != 0 && SMALL && TD > 0;  // Hessian assembly on the FP64 tensor pipe (2T <= 32, obstacles present)
  // compile-time (T, M) with DMMA assembly: the Hessian tiles stay in the accumulators and are factored there (nrmp_block_cholesky)
  constexpr bool kBlockChol = NB_NRMP_BLOCKCHOL != 0 && NB_NRMP_DMMA != 0 && SMALL && TT > 0 && MM > 0;
  constexpr int kNT = TT > 0 ? (2 * TT + 7) / 8 : 1, kTiles = kNT * (kNT + 1) / 2;
  // compile-time (T, M): the phases of the iteration run as fixed-trip, unrolled code with immediate shared-memory offsets; what
  // depends on the lane's row is a predicate, not a loop bound.  Every floating-point operation and its order are those of the
  // lane-bounded loops the generic instantiations run.
  constexpr bool kFixed = TT > 0;
  constexpr int kLaneUnroll = kFixed ? 8 : 1;

  // ---- carve this warp's workspace -------------------------------------------------------
  const int FT = T * (T + 1);                      // packed size of one component of F / G
  double* F = wsp;            wsp += 3 * FT;       // F[r][t][j] at r*FT + t(t+1) + j, j < 2(t+1)  (zero beyond)
  double* s0 = wsp;           wsp += 3 * T;        // s0[r][t]
  double* Hc = wsp;           wsp += nP;
  double* H = wsp;            wsp += (nU * (nU + 3)) >> 1;
  double* scratch = wsp;      wsp += nrmp_scratch_doubles(T, M);
  double* Gx = scratch;  double* Gy = scratch + FT;  // Hessian assembly (same packing as F)
  double* tmpk = scratch;                                // per-hinge values published for the per-step sums
  double* cv = wsp;           wsp += nU;
  double* x = wsp;            wsp += nU;
  double* rdU = wsp;          wsp += nU;
  double* dU = wsp;           wsp += nU;
  double* Dv = wsp;           wsp += T;
  double* dD = wsp;           wsp += T;
  double* rdD = wsp;          wsp += T;
  double* bD = wsp;           wsp += T;
  double* N00 = wsp;          wsp += T;
  double* N01 = wsp;          wsp += T;
  double* N11 = wsp;          wsp += T;
  double* n0 = wsp;           wsp += T;
  double* n1 = wsp;           wsp += T;
  double* iHDD = wsp;         wsp += T;
  double* e0 = wsp;           wsp += T;
  double* e1 = wsp;           wsp += T;
  double* qx = wsp;           wsp += T;
  double* qy = wsp;           wsp += T;
  double* cs = wsp;           wsp += mb;   // slacks of the box / rate / D rows
  double* cz = wsp;           wsp += mb;   // multipliers
  double* cds = wsp;          wsp += mb;
  double* cdz = wsp;          wsp += mb;   // holds rc on entry of a Newton solve, dz on exit
  float* cis = reinterpret_cast<float*>(wsp);  wsp += (mb + 1) / 2;  // inverse slacks
  float* fax_s = reinterpret_cast<float*>(wsp);
  float* fay_s = fax_s + TM;
  // setup-only linearisation data lives in the scratch region
  double* a02 = scratch;      double* a12 = scratch + T;  double* Bm = scratch + 2 * T;  double* Cm = scratch + 8 * T;
  double* gam_b = scratch + 11 * T;

  const float* ns = prm.nom_s + (size_t)b * 3 * T1;
  const float* nu = prm.nom_u + (size_t)b * 2 * T;
  const float* rs = prm.ref_s + (size_t)b * 3 * T1;
  const float* rus = prm.ref_us + (size_t)b * T;
  const bool omni = prm.kin == 2;
  const int rows_s = omni ? 2 : 3;
  const bool en_speed[2] = {isfinite(prm.speed[0]), isfinite(prm.speed[1])};
  const bool en_acce[2] = {isfinite(prm.acce[0]), isfinite(prm.acce[1])};
  const double rho = prm.ro, eta = (double)prm.eta;
  const double dlo = fmax((double)prm.d_min, 0.0), dhi = (double)prm.d_max;
  const bool dfix = TD > 0 && dhi == dlo;  // d_max == d_min: D is a constant, its bound rows and its Newton block drop out
  // rows of the shared-memory constraint block that are switched on: a row's class (box, rate, D) follows from k, and its control
  // component is k & 1 (the box and rate blocks start at even offsets and have even lengths nU and nR)
  auto enabled = [&](int k) -> bool {
    const bool c1 = (k & 1) != 0;
    return k < oRU ? (c1 ? en_speed[1] : en_speed[0]) : (k < oDU ? (c1 ? en_acce[1] : en_acce[0]) : !dfix);
  };
  int m_active = (dfix ? 0 : 2 * TD) + TM;
  for (int c = 0; c < 2; ++c) m_active += (en_speed[c] ? 2 * T : 0) + (en_acce[c] ? 2 * (T - 1) : 0);
  const double inv_m = 1.0 / (double)(m_active > 0 ? m_active : 1);

  // ---- 1. kinematics linearisation (robot.py:272-316, float32 tensor semantics) -------------
  const float fdt = (float)prm.dt;
  NB_LL(t, T) {
    const float v = nu[t];
    const float phi = (prm.kin == 2) ? nu[T + t] : ns[2 * T1 + t];
    const double snd = sin((double)phi), csd = cos((double)phi);
    const float snf = (float)snd, csf = (float)csd;
    a02[t] = omni ? 0.0 : (double)__fmul_rn(__fmul_rn(-v, fdt), snf);
    a12[t] = omni ? 0.0 : (double)__fmul_rn(__fmul_rn(v, fdt), csf);
    Cm[3 * t + 0] = (double)__fmul_rn(__fmul_rn(__fmul_rn(phi, v), snf), fdt);
    Cm[3 * t + 1] = (double)__fmul_rn(__fmul_rn(__fmul_rn(-phi, v), csf), fdt);
    Cm[3 * t + 2] = 0.0;
    double* Bt = Bm + 6 * t;  // row-major 3x2
    Bt[0] = (double)(float)(csd * prm.dt); Bt[1] = 0.0;
    Bt[2] = (double)(float)(snd * prm.dt); Bt[3] = 0.0;
    Bt[4] = 0.0; Bt[5] = 0.0;
    if (prm.kin == 0) {
      Bt[5] = (double)fdt;
    } else if (prm.kin == 1) {
      const float psi = nu[T + t];
      const double cp = cos((double)psi);
      const float den = (float)(prm.L * (cp * cp));
      Bt[4] = (double)(float)(tan((double)psi) * prm.dt / prm.L);
      Bt[5] = (double)__fdiv_rn(__fmul_rn(v, fdt), den);
      Cm[3 * t + 2] = (double)__fdiv_rn(__fmul_rn(__fmul_rn(-psi, v), fdt), den);
    } else {
      Bt[1] = (double)__fmul_rn(__fmul_rn(-v, snf), fdt);
      Bt[3] = (double)__fmul_rn(__fmul_rn(v, csf), fdt);
    }
    gam_b[t] = (double)__fmul_rn(prm.p_u, rus[t]);  // p_u * ref_us in float32 (nrmp.py:158)
  }
  __syncwarp();

  // ---- 2. free response s0 and sensitivities F (condensing) ---------------------------------
  if (lane == 0) {
    double px = ns[0], py = ns[T1], pth = ns[2 * T1];
    for (int t = 0; t < T; ++t) {
      const double nx = px + a02[t] * pth + Cm[3 * t], ny = py + a12[t] * pth + Cm[3 * t + 1], nth = pth + Cm[3 * t + 2];
      s0[t] = nx; s0[T + t] = ny; s0[2 * T + t] = nth;
      px = nx; py = ny; pth = nth;
    }
  }
  NB_LL(j, nU) {
    const int tj = j >> 1, cj = j & 1;
    double fx = 0, fy = 0, fth = 0;
    for (int t = 0; t < T; ++t) {
      if (t == tj) {
        fx = Bm[6 * t + cj]; fy = Bm[6 * t + 2 + cj]; fth = Bm[6 * t + 4 + cj];
      } else if (t > tj) {
        fx += a02[t] * fth; fy += a12[t] * fth;
      }
      if (t >= tj) { F[t * (t + 1) + j] = fx; F[FT + t * (t + 1) + j] = fy; F[2 * FT + t * (t + 1) + j] = fth; }
    }
  }
  __syncwarp();

  // ---- 3. quadratic cost 0.5 u^T Hc u + c^T u ------------------------------------------------
  double qd[3], qq[3];
  for (int r = 0; r < 3; ++r) {
    qq[r] = r < rows_s ? (double)prm.q[r] : 0.0;
    qd[r] = 2.0 * qq[r] * qq[r] + prm.bk;
  }
  const double pu = (double)prm.p_u;
  NB_LL(j, nU) {
    double acc = 0;
    for (int t = j >> 1; t < T; ++t)
      for (int r = 0; r < 3; ++r) {
        const double ga = (double)__fmul_rn(prm.q[r], rs[r * T1 + t + 1]);  // q_s * ref_s in float32
        const double g = 2.0 * qq[r] * ga + prm.bk * (double)ns[r * T1 + t + 1];
        acc += F[r * FT + t * (t + 1) + j] * (qd[r] * s0[r * T + t] - g);
      }
    if ((j & 1) == 0) acc += -2.0 * pu * gam_b[j >> 1];
    cv[j] = acc;
  }
  NB_LL(p, nP) {
    const int i = ptab[p] >> 8, j = ptab[p] & 255;
    double acc = 0;
    for (int t = i >> 1; t < T; ++t)
      for (int r = 0; r < 3; ++r) acc += qd[r] * F[r * FT + t * (t + 1) + i] * F[r * FT + t * (t + 1) + j];
    if (i == j && (i & 1) == 0) acc += 2.0 * pu * pu;
    Hc[p] = acc;
  }
  __syncwarp();  // the linearisation data in `scratch` is dead from here on

  // ---- 4. obstacle coefficients (nrmp.py:220-261), hinge rows owned by lanes -----------------------
  const int cnt = (prm.fa || M == 0) ? M : (prm.sel_count ? prm.sel_count[b] : 0);
  float hfx[HPL], hfy[HPL], his[HPL];
  double hs[HPL], hz[HPL], hds[HPL], hdz[HPL], hkk[HPL];
  int hts[HPL];     // horizon step of each owned hinge row
  double hih[HPL];  // 1/(rho + W) in FP64: the hinge elimination has to be exact for the Newton system to stay consistent
#pragma unroll
  for (int q_ = 0; q_ < HPL; ++q_) {
    const int k = lane + 32 * q_;
    hts[q_] = 0; hfx[q_] = 0.f; hfy[q_] = 0.f; hs[q_] = 1.0; hz[q_] = 0.0; hkk[q_] = 0.0;
    hds[q_] = hdz[q_] = 0.0; his[q_] = 0.f; hih[q_] = 0.0;
    if (k < TM) {
      const int t = k / M, mm = k - t * M;
      hts[q_] = t;
      float fx = 0.f, fy = 0.f, fbv = 0.f;
      if (prm.fa) {
        fx = prm.fa[((size_t)b * TM + k) * 2]; fy = prm.fa[((size_t)b * TM + k) * 2 + 1]; fbv = prm.fb[(size_t)b * TM + k];
      } else if (cnt > 0) {
        const int src = mm < cnt ? mm : 0;  // rows pn..M copy row 0 (nrmp.py:258-259)
        const size_t o = ((size_t)b * T1 + (t + 1)) * M + src;  // list entry t+1 (nrmp.py:244)
        fx = prm.sel_lam[o * 2]; fy = prm.sel_lam[o * 2 + 1];
        const float tmp = __fadd_rn(__fmul_rn(fx, prm.sel_pts[o * 2]), __fmul_rn(fy, prm.sel_pts[o * 2 + 1]));
        float muh = 0.f;
        for (int e = 0; e < prm.E; ++e) muh = fmaf(prm.sel_mu[o * prm.E + e], prm.h[e], muh);
        fbv = __fadd_rn(tmp, muh);
      }
      hfx[q_] = fx; hfy[q_] = fy;
      fax_s[k] = fx; fay_s[k] = fy;
      hkk[q_] = (double)fbv - ((double)fx * s0[t] + (double)fy * s0[T + t]);  // hinge argument at u = 0, without D_t
    }
  }

  // gradient scale of the program: the dual-residual test is relative to it.  An environment whose cost gradient is O(1e3)
  // cannot reach an absolute 1e-8 in FP64 once the barrier weights are large; its residual then idles at ~2e-8 while the gap is
  // driven to 1e-16 and the factorisation finally breaks (seen on 5 % of the C5 problems and on C4 env 934 in the CPU oracle).
  double res_scale = 1.0;
  {
    double m = 0.0;
    NB_LL(i, nU) m = fmax(m, fabs(cv[i]));
#pragma unroll
    for (int q_ = 0; q_ < HPL; ++q_)
      if (lane + 32 * q_ < TM) m = fmax(m, rho * fabs(hkk[q_]));
    res_scale = fmax(1.0, warp_max(m));
  }
  const double res_tol = 1e-8 * res_scale;

  // ---- 5. strictly feasible start: cold (u = 0, D mid-range) or warm (previous solve of this environment) ------
  int stat = 0;
  if (TD > 0 && dhi < dlo) stat |= 4;
  for (int c = 0; c < 2; ++c) {
    if (en_speed[c] && !(prm.speed[c] > 0)) stat |= 4;
    if (en_acce[c] && !(prm.acce[c] > 0)) stat |= 4;
  }
  const size_t warm_floats = nrmp_warm_floats(T, M);
  float* wrec = prm.warm ? prm.warm + (size_t)b * warm_floats : nullptr;
  const bool try_warm = wrec != nullptr && prm.warm_valid[b] == 1 && stat == 0;
  const double dmid = 0.5 * (dlo + dhi);
  // warm start constants, measured on C4 / C2 problem sequences (DESIGN.md 3.2): pull-back towards the centre, complementarity
  // floor mu0, cap kKappa * mu0 on s z (an uncapped multiplier of a row that is no longer active leaves Mehrotra's iteration in
  // a 2-cycle: C4 envs 1507 / 2530), margin of the hinge rows
  constexpr double kTheta = 0.05, kMu0 = 1e-2, kDw = 0.03, kKappa = 100.0;
  int it = 0, it_total = 0;
  bool converged = false, banned = false, have_factor = false;
  double invd0 = 0.0, invd1 = 0.0;  // 1 / diag(L) of the rows this lane owns (last factorisation)
#pragma unroll 1
  for (int attempt = 0; attempt < 2; ++attempt) {  // attempt 0: warm if allowed; attempt 1: cold restart of a warm start that went wrong
  const bool warm = try_warm && attempt == 0;
  bool restart = false;
  stat &= ~3;
  __syncwarp();  // a restart re-initialises shared state the abandoned attempt was still reading (ordered only by shuffles)
  NB_LL(i, nU) x[i] = warm ? (1.0 - kTheta) * (double)wrec[i] : 0.0;
  NB_LL(t, TD) Dv[t] = dfix ? dlo : (warm ? (1.0 - kTheta) * (double)wrec[nU + t] + kTheta * dmid : dmid);
  __syncwarp();
  NB_LL(i, nU) {
    const int c = i & 1;
    const double xi = x[i];
    const double su = en_speed[c] ? prm.speed[c] - xi : 1.0, sl = en_speed[c] ? prm.speed[c] + xi : 1.0;
    cs[oBU + i] = su; cs[oBL + i] = sl;
    double zu = en_speed[c] ? (warm ? kMu0 : 1.0) / su : 0.0, zl = en_speed[c] ? (warm ? kMu0 : 1.0) / sl : 0.0;
    if (warm && en_speed[c]) {
      zu = fmin(fmax(zu, (double)wrec[nU + TD + oBU + i]), kKappa * zu); zl = fmin(fmax(zl, (double)wrec[nU + TD + oBL + i]), kKappa * zl);
    }
    cz[oBU + i] = zu; cz[oBL + i] = zl;
    if (i < nR) {
      const double dd = x[i + 2] - xi;
      const double ru = en_acce[c] ? prm.acce[c] - dd : 1.0, rl = en_acce[c] ? prm.acce[c] + dd : 1.0;
      cs[oRU + i] = ru; cs[oRL + i] = rl;
      double yu = en_acce[c] ? (warm ? kMu0 : 1.0) / ru : 0.0, yl = en_acce[c] ? (warm ? kMu0 : 1.0) / rl : 0.0;
      if (warm && en_acce[c]) {
        yu = fmin(fmax(yu, (double)wrec[nU + TD + oRU + i]), kKappa * yu); yl = fmin(fmax(yl, (double)wrec[nU + TD + oRL + i]), kKappa * yl);
      }
      cz[oRU + i] = yu; cz[oRL + i] = yl;
    }
  }
  NB_LL(t, TD) {
    if (dfix) {
      cs[oDU + t] = cs[oDL + t] = 1.0; cz[oDU + t] = cz[oDL + t] = 0.0;
    } else {
      const double su = dhi - Dv[t], sl = Dv[t] - dlo;
      cs[oDU + t] = su; cs[oDL + t] = sl;
      double zu = (warm ? kMu0 : 1.0) / su, zl = (warm ? kMu0 : 1.0) / sl;
      if (warm) { zu = fmin(fmax(zu, (double)wrec[nU + TD + oDU + t]), kKappa * zu); zl = fmin(fmax(zl, (double)wrec[nU + TD + oDL + t]), kKappa * zl); }
      cz[oDU + t] = zu; cz[oDL + t] = zl;
    }
    // position offset F x of the start (zero when cold): qx / qy are free until the first Newton solve
    double ax = 0, ay = 0;
    if (warm) {
      const double* fxp = F + t * (t + 1);
      const double* fyp = fxp + FT;
      for (int i = 0; i < 2 * (t + 1); ++i) { ax += fxp[i] * x[i]; ay += fyp[i] * x[i]; }
    }
    qx[t] = ax; qy[t] = ay;
  }
  __syncwarp();
#pragma unroll
  for (int q_ = 0; q_ < HPL; ++q_) {
    const int k = lane + 32 * q_;
    if (k < TM) {
      const int t = hts[q_];
      const double r = Dv[t] + hkk[q_] - ((double)hfx[q_] * qx[t] + (double)hfy[q_] * qy[t]);
      // s = z/rho - r > 0 needs z > rho r; rows far on the inactive side may start with a small multiplier
      double z;
      if (warm) {
        const double zlo = fmax(rho * fmax(r + kDw, 0.0), kMu0 / fmax(-r, kDw));
        z = fmax(fmin((double)wrec[nU + TD + mb + k], fmax(kKappa * kMu0 / fmax(-r, kDw), zlo)), zlo);
      }
      else z = fmax(rho * fmax(r + 0.1, 0.0), 1.0 / fmax(-r, 0.1));
      hz[q_] = z; hs[q_] = z / rho - r;
    }
  }
  __syncwarp();
  NB_PHASE(0);

  // ---- 6. interior point iterations -------------------------------------------------------------
  converged = false;
  bool accept_gap = false;
  have_factor = false;
  if (stat == 0) {
#pragma unroll 1
    for (it = 0; it < prm.max_ipm_iter; ++it) {
      // (a) dual residual, gap
#pragma unroll
      for (int q_ = 0; q_ < HPL; ++q_) {
        const int k = lane + 32 * q_;
        if (k < TM) tmpk[k] = hz[q_];
      }
      __syncwarp();
      NB_LW(t, TD) {
        double gx = 0, gy = 0, sz = 0;
        for (int mm = 0; mm < M; ++mm) {
          const int k = t * M + mm;
          const double zr = tmpk[k];
          gx += zr * (double)fax_s[k]; gy += zr * (double)fay_s[k]; sz += zr;
        }
        e0[t] = gx; e1[t] = gy;  // (e0/e1 carry g_t here; rewritten inside the Newton solve)
        rdD[t] = -eta + cz[oDU + t] - cz[oDL + t] + sz;
      }
      __syncwarp();
      double res = 0.0, gsum = 0.0;
      NB_LW(i, nU) {
        double acc = cv[i];
        if constexpr (kFixed) {
          // row i of the packed lower triangle (Hc[i(i+1)/2 + j], j <= i), then column i below the diagonal (Hc[j(j+1)/2 + i],
          // j > i): the two parts are independent FMA chains
          const double* hp = Hc + i * (i + 1) / 2;
          double accq = 0.0;
#pragma unroll
          for (int j = 0; j < nU; ++j) {
            if (j <= i) acc += hp[j] * x[j];
            else accq += Hc[j * (j + 1) / 2 + i] * x[j];
          }
          acc += accq;
        } else {
          const double* hp = Hc + i * (i + 1) / 2;  // row i of the packed lower triangle, then column i below the diagonal
          const double* hq = hp + i + i + 1;        // element (i+1, i)
          double accq = 0.0;                        // the two parts are independent FMA chains
#pragma unroll 2
          for (int j = 0; j <= i; ++j) acc += hp[j] * x[j];
#pragma unroll 2
          for (int j = i + 1; j < nU; ++j) { accq += *hq * x[j]; hq += j + 1; }
          acc += accq;
        }
        acc += cz[oBU + i] - cz[oBL + i];
        if (i >= 2) acc += cz[oRU + i - 2] - cz[oRL + i - 2];
        if (i < nR) acc -= cz[oRU + i] - cz[oRL + i];
        if (TD > 0) {
          double accy = 0.0;
          if constexpr (kFixed) {
#pragma unroll
            for (int t = 0; t < T; ++t)  // F_t has columns [0, 2t + 2)
              if (i < 2 * t + 2) { acc -= F[t * (t + 1) + i] * e0[t]; accy -= F[FT + t * (t + 1) + i] * e1[t]; }
          } else {
            const double* fxp = F + (i >> 1) * ((i >> 1) + 1) + i;
            const double* fyp = fxp + FT;
#pragma unroll 2
            for (int t = i >> 1; t < T; ++t) { acc -= fxp[0] * e0[t]; accy -= fyp[0] * e1[t]; fxp += 2 * (t + 1); fyp += 2 * (t + 1); }
          }
          acc += accy;
        }
        rdU[i] = acc;
        res = fmax(res, fabs(acc));
      }
      if (!dfix) NB_LW(t, TD) res = fmax(res, fabs(rdD[t]));
      NB_LW(k, mb) if (enabled(k)) gsum += cs[k] * cz[k];
#pragma unroll
      for (int q_ = 0; q_ < HPL; ++q_)
        if (lane + 32 * q_ < TM) gsum += hs[q_] * hz[q_];
      res = warp_max(res);
      const double gap = warp_sum(gsum) * inv_m;
      if (!(gap == gap) || !(res == res)) { stat |= 2; break; }
      // differentiable mode: the converged iterate goes through (b)-(d) once more so that the factor that is saved for the
      // adjoint belongs to the final point
      const bool finishing = gap < prm.gap_tol && res < res_tol;
      if (finishing && prm.adj_save == nullptr) { converged = true; break; }
      // a warm start that is not well on its way by iteration 12 (gap still above 1e-5; a healthy one is below 1e-8 there) is
      // abandoned for a cold start -- rare (<1 % on C4), but one 60-iteration straggler would set the duration of the launch
      if (warm && ((it == 12 && gap > 1e-5) || (it == prm.warm_check_it && gap > prm.warm_check_gap))) { restart = true; break; }
      accept_gap = gap < 1e-9 && res < 10.0 * res_tol;  // good enough to keep if the next factorisation fails in rounding noise
      NB_PHASE(1);

      // (b) barrier weights; hinge rows publish omega for the per-step reductions
      __syncwarp();
      // Differentiable mode, final pass: the factor that is saved for the adjoint is that of the active-set system.  A row whose
      // multiplier exceeds its slack is active and held by W = 1e9; any other row keeps its barrier weight W = z/s (< 1).  With
      // W = z/s = 1e13+ the information about the cost Hessian along an active RATE constraint (W (e_{i+2} - e_i)(e_{i+2} - e_i)'
      // couples two controls) survives only through the cancellation of 1e14-sized entries: measured gradient errors of 1e-2 (C5,
      // acceleration-limited) that grew to 3e-1 with a tighter gap; a pinned direction held by 1e9 instead of infinity moves the
      // result by 1e-7.  A weight that grows with z instead (z^2 / 1e-10) leaves a row held by a small multiplier soft: z = 4e-4
      // gave W = 1.6e3 and a 3.6e-2 error of the chain gradient (C4 `obstacles`, env 141 of 1024).
      NB_LW(k, mb) {
        if (finishing && enabled(k)) {
          const double sk = cs[k], zk = cz[k];
          cis[k] = (float)(zk > sk ? 1e9 / zk : 1.0 / sk);
        } else {
          cis[k] = rcpf(cs[k]);
        }
      }
#pragma unroll
      for (int q_ = 0; q_ < HPL; ++q_) {
        const int k = lane + 32 * q_;
        if (k < TM) {
          his[q_] = finishing ? (float)(hz[q_] > hs[q_] ? 1e9 / hz[q_] : 1.0 / hs[q_]) : rcpf(hs[q_]);
          const double Wr = hz[q_] * (double)his[q_];
          hih[q_] = rcp64(rho + Wr);
          tmpk[k] = Wr * rho * hih[q_];  // omega: the row's weight in the reduced Hessian (bounded by rho)
        }
      }
      __syncwarp();
      NB_LW(t, TD) {
        double a00 = 0, a01 = 0, a11 = 0, b0 = 0, b1 = 0, nn = 0;
        for (int mm = 0; mm < M; ++mm) {
          const int k = t * M + mm;
          const double om = tmpk[k], fx = (double)fax_s[k], fy = (double)fay_s[k];
          const double ofx = om * fx, ofy = om * fy;
          a00 += ofx * fx; a01 += ofx * fy; a11 += ofy * fy; b0 += ofx; b1 += ofy; nn += om;
        }
        const double hdd = nn + cz[oDU + t] * (double)cis[oDU + t] + cz[oDL + t] * (double)cis[oDL + t];
        const double ih = dfix ? 0.0 : rcp64(hdd);  // fixed D: no D block, dD = 0
        iHDD[t] = ih; n0[t] = b0; n1[t] = b1;
        const double m00 = a00 - b0 * b0 * ih, m01 = a01 - b0 * b1 * ih, m11 = a11 - b1 * b1 * ih;
        if (kDmma) {
          // N_t = R'R (2x2 Cholesky; N_t is positive semidefinite by Cauchy-Schwarz, hdd >= sum omega): the Hessian update
          // sum_t F_t' N_t F_t becomes V'V with V_t = R_t F_t, a plain Gram matrix for the tensor pipe
          double r00 = 0.0, r01 = 0.0, r11 = 0.0;
          if (m00 > 1e-30) { const double ir = rsqrt64(m00); r00 = m00 * ir; r01 = m01 * ir; }
          const double v = fma(-r01, r01, m11);
          if (v > 1e-30) r11 = v * rsqrt64(v);
          N00[t] = r00; N01[t] = r01; N11[t] = r11;
        } else {
          N00[t] = m00; N01[t] = m01; N11[t] = m11;
        }
      }
      __syncwarp();
      NB_PHASE(2);
      double tl0[kTiles], tl1[kTiles];  // kBlockChol: the Hessian tiles of (c), factored in place by (d)
      if (kDmma) {
        // V (packed like F, in the Gx | Gy scratch): row 2t = r00 Fx_t + r01 Fy_t, row 2t+1 = r11 Fy_t
        NB_LW(j, nU) {
          if constexpr (kFixed) {
#pragma unroll
            for (int t = 0; t < T; ++t) {
              if (j < 2 * t + 2) {
                const int o = t * (t + 1) + j;
                const double fx = F[o], fy = F[FT + o];
                Gx[o] = N00[t] * fx + N01[t] * fy;
                Gy[o] = N11[t] * fy;
              }
            }
          } else {
            int o = (j >> 1) * ((j >> 1) + 1) + j;
#pragma unroll 2
            for (int t = j >> 1; t < T; ++t) {
              const double fx = F[o], fy = F[FT + o];
              Gx[o] = N00[t] * fx + N01[t] * fy;
              Gy[o] = N11[t] * fy;
              o += 2 * (t + 1);
            }
          }
        }
        __syncwarp();
        // (c) reduced Hessian = Hc + V'V + bound terms: 8x8 tiles of the lower triangle on the FP64 tensor pipe (DMMA m8n8k4),
        //     k-steps whose four rows of V are structurally zero in the tile's columns are skipped (T = 10: 14 DMMAs)
        const int q = lane & 3, g = lane >> 2;
        const int nT = (nU + 7) >> 3;
#pragma unroll
        for (int I = 0; I < (TT > 0 ? (2 * TT + 7) / 8 : 4); ++I) {
          if (I >= nT) break;
          const int i0 = 8 * I, ia = i0 + g;
#pragma unroll
          for (int J = 0; J <= I; ++J) {
            const int j0 = 8 * J, jb = j0 + g;
            double c0 = 0.0, c1 = 0.0;
#pragma unroll
            for (int k0 = 0; k0 < (TT > 0 ? 2 * TT : 32); k0 += 4) {
              if (k0 >= nU) break;
              if (2 * (((k0 + 3) >> 1) + 1) <= i0) continue;  // rows k0..k0+3 have no entries in columns >= i0
              const int k = k0 + q, t = k >> 1;
              const int lim = k < nU ? 2 * t + 2 : 0;  // row k = 2t + c of V has columns [0, 2t + 2)
              const double* vr = Gx + (k & 1) * FT + t * (t + 1);
              const double a = ia < lim ? vr[ia] : 0.0;
              const double b = I == J ? a : (jb < lim ? vr[jb] : 0.0);
              dmma884(c0, c1, a, b);
            }
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int i = ia, j = j0 + 2 * q + e;
              if constexpr (kBlockChol) (e ? tl1 : tl0)[I * (I + 1) / 2 + J] = i == j ? 1.0 : 0.0;  // padding: identity; diagonal tiles: 0 above
              if (i < nU && j <= i) {
                double acc = Hc[(i * (i + 1) >> 1) + j] + (e ? c1 : c0);
                if (i == j) {
                  acc += cz[oBU + i] * (double)cis[oBU + i] + cz[oBL + i] * (double)cis[oBL + i];
                  if (i >= 2) acc += cz[oRU + i - 2] * (double)cis[oRU + i - 2] + cz[oRL + i - 2] * (double)cis[oRL + i - 2];
                  if (i < nR) acc += cz[oRU + i] * (double)cis[oRU + i] + cz[oRL + i] * (double)cis[oRL + i];
                } else if (i == j + 2) {
                  acc -= cz[oRU + j] * (double)cis[oRU + j] + cz[oRL + j] * (double)cis[oRL + j];
                }
                if constexpr (kBlockChol) (e ? tl1 : tl0)[I * (I + 1) / 2 + J] = acc;
                else H[hrow(i) + j] = acc;
              }
            }
          }
        }
      } else {
      if (TD > 0) {
        NB_LL(j, nU) {
          int o = (j >> 1) * ((j >> 1) + 1) + j;
#pragma unroll 2
          for (int t = j >> 1; t < T; ++t) {
            const double fx = F[o], fy = F[FT + o];
            Gx[o] = N00[t] * fx + N01[t] * fy;
            Gy[o] = N01[t] * fx + N11[t] * fy;
            o += 2 * (t + 1);
          }
        }
        __syncwarp();
      }
      // (c) reduced Hessian, lower triangle
      NB_LL(p, nP) {
        const int i = ptab[p] >> 8, j = ptab[p] & 255;
        double acc = Hc[p];
        if (TD > 0) {
          int o = (i >> 1) * ((i >> 1) + 1);  // row t = i/2 of the packed layout; j <= i < 2(t+1) so both columns exist
          double accy = 0.0;
#pragma unroll 2
          for (int t = i >> 1; t < T; ++t) {
            acc += F[o + i] * Gx[o + j];
            accy += F[FT + o + i] * Gy[o + j];
            o += 2 * (t + 1);
          }
          acc += accy;
        }
        if (i == j) {
          acc += cz[oBU + i] * (double)cis[oBU + i] + cz[oBL + i] * (double)cis[oBL + i];
          if (i >= 2) acc += cz[oRU + i - 2] * (double)cis[oRU + i - 2] + cz[oRL + i - 2] * (double)cis[oRL + i - 2];
          if (i < nR) acc += cz[oRU + i] * (double)cis[oRU + i] + cz[oRL + i] * (double)cis[oRL + i];
        } else if (i == j + 2) {
          acc -= cz[oRU + j] * (double)cis[oRU + j] + cz[oRL + j] * (double)cis[oRL + j];
        }
        H[hrow(i) + j] = acc;
      }
      }
      __syncwarp();
      NB_PHASE(3);
      // (d) Cholesky.  kBlockChol: blocked, on the tiles of (c) (nrmp_block_cholesky).  Otherwise left-looking; lane owns rows
      //     lane, lane+32; inverse diagonal in registers.  SMALL: two columns per step (nU = 2T is even) -- row i is read once
      //     for both dot products, which are two independent FMA chains; the second column then takes the rank-1 correction
      //     of the first.
      bool bad = false;
#if NB_NRMP_CHOL_TWICE
      // timing only (NB_NRMP_CHOL_TWICE): (d) runs twice on the same Hessian -- the unblocked form restores H from `scratch`
      // (dead here) in between; results and iteration counts are unchanged, so the difference in launch time is the cost of
      // one factorisation (plus the copies)
      if (!kBlockChol) {
        NB_LL(p, nP) scratch[p] = H[hrow(ptab[p] >> 8) + (ptab[p] & 255)];
        __syncwarp();
      }
#pragma unroll 1
      for (int rep = 0; rep < 2; ++rep) {
      if (rep == 1 && !kBlockChol) {
        NB_LL(p, nP) H[hrow(ptab[p] >> 8) + (ptab[p] & 255)] = scratch[p];
        __syncwarp();
      }
      bad = false;
#endif
      invd0 = 0.0; invd1 = 0.0;
      if constexpr (kBlockChol) {
        double w0[kTiles], w1[kTiles];
#pragma unroll
        for (int i = 0; i < kTiles; ++i) { w0[i] = tl0[i]; w1[i] = tl1[i]; }
        bad = !nrmp_block_cholesky<kNT, 2 * TT>(w0, w1, H, invd0, lane);
      } else if (SMALL) {
#pragma unroll(kUnrollCholK)
        for (int k = 0; k < nU; k += 2) {
          const double* rowk = H + hrow(k);
          const double* rowk1 = H + hrow(k + 1);
          const bool in0 = lane >= k && lane < nU, in1 = lane > k && lane < nU;
          double a0 = 0.0, a1 = 0.0;
          if (in0) {
            const double* rowi = H + hrow(lane);
            a0 = rowi[k];
            if (in1) a1 = rowi[k + 1];
#pragma unroll(kUnrollCholP)
            for (int p = 0; p < k; ++p) {
              const double v = rowi[p];
              a0 -= v * rowk[p];
              a1 -= v * rowk1[p];
            }
          }
          const double d0 = __shfl_sync(0xffffffffu, a0, k);
          if (!(d0 > 0.0)) { bad = true; break; }
          const double ild0 = rsqrt64(d0);
          const double l0 = a0 * ild0;                            // L[lane][k]
          const double l10 = __shfl_sync(0xffffffffu, l0, k + 1);  // L[k+1][k]
          a1 -= l0 * l10;
          const double d1 = __shfl_sync(0xffffffffu, a1, k + 1);
          if (!(d1 > 0.0)) { bad = true; break; }
          const double ild1 = rsqrt64(d1);
          if (lane == k) invd0 = ild0;
          if (lane == k + 1) invd0 = ild1;
          if (in0) H[hrow(lane) + k] = l0;
          if (in1) H[hrow(lane) + k + 1] = a1 * ild1;
          __syncwarp();
        }
      } else {
#pragma unroll 1
        for (int k = 0; k < nU; ++k) {
          double acc0 = 0.0, acc1 = 0.0;
          const int i0 = lane, i1 = lane + 32;
          const double* rowk = H + hrow(k);
          if (i0 >= k && i0 < nU) {
            const double* rowi = H + hrow(i0);
            acc0 = rowi[k];
#pragma unroll 4
            for (int p = 0; p < k; ++p) acc0 -= rowi[p] * rowk[p];
          }
          if (i1 >= k && i1 < nU) {
            const double* rowi = H + hrow(i1);
            acc1 = rowi[k];
#pragma unroll 4
            for (int p = 0; p < k; ++p) acc1 -= rowi[p] * rowk[p];
          }
          const double d = __shfl_sync(0xffffffffu, k < 32 ? acc0 : acc1, k & 31);
          if (!(d > 0.0)) { bad = true; break; }
          const double ild = rsqrt64(d);
          if (i0 == k) invd0 = ild;
          if (i1 == k) invd1 = ild;
          if (i0 >= k && i0 < nU) H[hrow(i0) + k] = acc0 * ild;
          if (i1 >= k && i1 < nU) H[hrow(i1) + k] = acc1 * ild;
          __syncwarp();
        }
      }
#if NB_NRMP_CHOL_TWICE
      }
#endif
      NB_PHASE(4);
      if (bad) {  // H lost definiteness: at barrier weights of 1e13+ that is rounding, and the iterate is already the optimum
        if (accept_gap) converged = true;
        else stat |= 2;
        break;
      }

      if (finishing) { converged = true; have_factor = true; break; }
      // (e) predictor (pass 0) and corrector (pass 1) share one Newton body
      NB_LW(k, mb) cdz[k] = enabled(k) ? -cs[k] * cz[k] : 0.0;
#pragma unroll
      for (int q_ = 0; q_ < HPL; ++q_) hdz[q_] = -hs[q_] * hz[q_];
      double alpha = 1.0;
#pragma unroll 1
      for (int pass = 0; pass < 2; ++pass) {
        __syncwarp();
        // hinge rows: v = rc / s and their right-hand-side contribution y = -(rho / (rho + W)) v
        double hv[HPL];
#pragma unroll
        for (int q_ = 0; q_ < HPL; ++q_) {
          const int k = lane + 32 * q_;
          hv[q_] = 0.0;
          if (k < TM) {
            hv[q_] = hdz[q_] * (double)his[q_];
            tmpk[k] = -rho * hih[q_] * hv[q_];
          }
        }
        __syncwarp();
        NB_LW(t, TD) {
          double Y0 = 0, Y1 = 0, Ys = 0;
          for (int mm = 0; mm < M; ++mm) {
            const int k = t * M + mm;
            const double y = tmpk[k];
            Y0 += y * (double)fax_s[k]; Y1 += y * (double)fay_s[k]; Ys += y;
          }
          const double vdu = cdz[oDU + t] * (double)cis[oDU + t], vdl = cdz[oDL + t] * (double)cis[oDL + t];
          const double bb = -rdD[t] - (vdu - vdl) + Ys;
          bD[t] = bb;
          e0[t] = -Y0 + n0[t] * bb * iHDD[t];
          e1[t] = -Y1 + n1[t] * bb * iHDD[t];
        }
        __syncwarp();
        // right-hand side rows in registers, then L y = b, L^T x = y with shuffles
        double r0 = 0.0, r1 = 0.0;
#pragma unroll
        for (int sl = 0; sl < (SMALL ? 1 : 2); ++sl) {
          const int i = lane + 32 * sl;
          if (i < nU) {
            double acc = -rdU[i] - (cdz[oBU + i] * (double)cis[oBU + i] - cdz[oBL + i] * (double)cis[oBL + i]);
            if (i >= 2) acc -= cdz[oRU + i - 2] * (double)cis[oRU + i - 2] - cdz[oRL + i - 2] * (double)cis[oRL + i - 2];
            if (i < nR) acc += cdz[oRU + i] * (double)cis[oRU + i] - cdz[oRL + i] * (double)cis[oRL + i];
            if (TD > 0) {
              double accy = 0.0;
              if constexpr (kFixed) {
#pragma unroll
                for (int t = 0; t < T; ++t)  // F_t has columns [0, 2t + 2)
                  if (i < 2 * t + 2) { acc += F[t * (t + 1) + i] * e0[t]; accy += F[FT + t * (t + 1) + i] * e1[t]; }
              } else {
                const double* fxp = F + (i >> 1) * ((i >> 1) + 1) + i;
                const double* fyp = fxp + FT;
#pragma unroll 2
                for (int t = i >> 1; t < T; ++t) { acc += fxp[0] * e0[t]; accy += fyp[0] * e1[t]; fxp += 2 * (t + 1); fyp += 2 * (t + 1); }
              }
              acc += accy;
            }
            if (sl == 0) r0 = acc; else r1 = acc;
          }
        }
        if (SMALL) {
          // r0 stays the running residual of this lane's row (no select per step: row k is final when step k reads it), the
          // scaling by 1 / L_kk rides on the broadcast; with compile-time T both loops unroll into shuffle + predicated FMA
          const double* rowl = H + hrow(lane < nU ? lane : 0);  // L[lane][k], k < lane (idle lanes read row 0, results unused)
#pragma unroll(kUnrollSolve)
          for (int k = 0; k < nU; ++k) {
            const double yk = __shfl_sync(0xffffffffu, r0 * invd0, k);
            if (lane > k) r0 = fma(-rowl[k], yk, r0);
          }
          r0 *= invd0;  // y = L^-1 b
          const double* coll = H + lane;  // L[k][lane], k > lane
#pragma unroll(kUnrollSolve)
          for (int k = nU - 1; k >= 0; --k) {
            const double xk = __shfl_sync(0xffffffffu, r0 * invd0, k);
            if (lane < k) r0 = fma(-coll[hrow(k)], xk, r0);
          }
          r0 *= invd0;  // x = L^-T y
        } else {
#pragma unroll 1
          for (int k = 0; k < nU; ++k) {
            const double mine = k < 32 ? r0 * invd0 : r1 * invd1;
            const double yk = __shfl_sync(0xffffffffu, mine, k & 31);
            if (lane == (k & 31)) { if (k < 32) r0 = yk; else r1 = yk; }
            if (lane > k && lane < nU) r0 -= H[hrow(lane) + k] * yk;
            if (lane + 32 > k && lane + 32 < nU) r1 -= H[hrow(lane + 32) + k] * yk;
          }
#pragma unroll 1
          for (int k = nU - 1; k >= 0; --k) {
            const double mine = k < 32 ? r0 * invd0 : r1 * invd1;
            const double xk = __shfl_sync(0xffffffffu, mine, k & 31);
            if (lane == (k & 31)) { if (k < 32) r0 = xk; else r1 = xk; }
            if (lane < k) r0 -= H[hrow(k) + lane] * xk;
            if (lane + 32 < k) r1 -= H[hrow(k) + lane + 32] * xk;
          }
        }
        if (lane < nU) dU[lane] = r0;
        if (!SMALL && lane + 32 < nU) dU[lane + 32] = r1;
        __syncwarp();
        NB_LW(t, TD) {
          double ax = 0, ay = 0;
          const double* fxp = F + t * (t + 1);
          const double* fyp = fxp + FT;
          if constexpr (kFixed) {
#pragma unroll
            for (int i = 0; i < nU; ++i)
              if (i < 2 * t + 2) { ax += fxp[i] * dU[i]; ay += fyp[i] * dU[i]; }
          } else {
#pragma unroll 2
            for (int i = 0; i < 2 * (t + 1); ++i) {
              ax += fxp[i] * dU[i];
              ay += fyp[i] * dU[i];
            }
          }
          qx[t] = ax; qy[t] = ay;
          dD[t] = (bD[t] + n0[t] * ax + n1[t] * ay) * iHDD[t];
        }
        __syncwarp();
        // steps of slacks / multipliers, and the largest relative decrease (for the step length)
        float ratio = 0.f;
#pragma unroll
        for (int q_ = 0; q_ < HPL; ++q_) {
          const int k = lane + 32 * q_;
          if (k < TM) {
            const int t = hts[q_];
            const double Jdx = dD[t] - ((double)hfx[q_] * qx[t] + (double)hfy[q_] * qy[t]);
            const double Wr = hz[q_] * (double)his[q_];
            const double dw = hih[q_] * (hv[q_] + Wr * Jdx);  // step of the eliminated w = z / rho
            hds[q_] = dw - Jdx;   // s = z/rho - r stays exact: ds = dz/rho - J dx
            hdz[q_] = rho * dw;
            ratio = fmaxf(ratio, fmaxf(-(float)hds[q_] * his[q_], -(float)hdz[q_] * rcpf(hz[q_])));
          }
        }
        NB_LW(i, nU) {
          const double d = dU[i];
          cdz[oBU + i] = (cdz[oBU + i] + cz[oBU + i] * d) * (double)cis[oBU + i]; cds[oBU + i] = -d;
          cdz[oBL + i] = (cdz[oBL + i] - cz[oBL + i] * d) * (double)cis[oBL + i]; cds[oBL + i] = d;
          if (i < nR) {
            const double dd = dU[i + 2] - d;
            cdz[oRU + i] = (cdz[oRU + i] + cz[oRU + i] * dd) * (double)cis[oRU + i]; cds[oRU + i] = -dd;
            cdz[oRL + i] = (cdz[oRL + i] - cz[oRL + i] * dd) * (double)cis[oRL + i]; cds[oRL + i] = dd;
          }
        }
        NB_LW(t, TD) {
          const double d = dD[t];
          cdz[oDU + t] = (cdz[oDU + t] + cz[oDU + t] * d) * (double)cis[oDU + t]; cds[oDU + t] = -d;
          cdz[oDL + t] = (cdz[oDL + t] - cz[oDL + t] * d) * (double)cis[oDL + t]; cds[oDL + t] = d;
        }
        __syncwarp();
        NB_LW(k, mb) {
          if (!enabled(k)) continue;
          ratio = fmaxf(ratio, fmaxf(-(float)cds[k] * cis[k], -(float)cdz[k] * rcpf(cz[k])));
        }
        ratio = warp_maxf(ratio);
        if (pass == 0) {
          const double amax = ratio > 1.0f ? 1.0 / (double)ratio : 1.0;  // largest step <= 1 keeping s, z >= 0
          double ga = 0.0;
          NB_LW(k, mb) if (enabled(k)) ga += (cs[k] + amax * cds[k]) * (cz[k] + amax * cdz[k]);
#pragma unroll
          for (int q_ = 0; q_ < HPL; ++q_)
            if (lane + 32 * q_ < TM) ga += (hs[q_] + amax * hds[q_]) * (hz[q_] + amax * hdz[q_]);
          const double sr = fmax(warp_sum(ga) * inv_m, 0.0) / gap;
          const double smu = sr * sr * sr * gap;  // sigma * mu
          NB_LW(k, mb) cdz[k] = enabled(k) ? (-cs[k] * cz[k] + smu - cds[k] * cdz[k]) : 0.0;
#pragma unroll
          for (int q_ = 0; q_ < HPL; ++q_) hdz[q_] = -hs[q_] * hz[q_] + smu - hds[q_] * hdz[q_];
        } else {
          alpha = ratio > 0.995f ? 0.995 / (double)ratio : 1.0;
        }
      }
      NB_LW(i, nU) x[i] += alpha * dU[i];
      NB_LW(t, TD) Dv[t] += alpha * dD[t];
      NB_LW(k, mb) if (enabled(k)) { cs[k] += alpha * cds[k]; cz[k] += alpha * cdz[k]; }
#pragma unroll
      for (int q_ = 0; q_ < HPL; ++q_) {
        if (lane + 32 * q_ < TM) { hs[q_] += alpha * hds[q_]; hz[q_] += alpha * hdz[q_]; }
      }
      __syncwarp();
      NB_PHASE(5);
    }
    if (!converged && !(stat & 2) && !restart) stat |= 1;
  }
  it_total += it;
  if (warm && (restart || (stat & 3))) { banned = true; continue; }  // cold restart
  break;
  }  // attempt
  it = it_total;
  if (wrec) {  // the next PAN iteration of this environment starts from here (only from a converged solve)
    __syncwarp();
    if (stat == 0) {
      NB_LL(i, nU) wrec[i] = (float)x[i];
      NB_LL(t, TD) wrec[nU + t] = (float)Dv[t];
      NB_LL(k, mb) wrec[nU + TD + k] = (float)cz[k];
#pragma unroll
      for (int q_ = 0; q_ < HPL; ++q_)
        if (lane + 32 * q_ < TM) wrec[nU + TD + mb + lane + 32 * q_] = (float)hz[q_];
    }
    // 2 = this environment's warm start failed once in this forward(): its remaining solves start cold
    if (lane == 0) prm.warm_valid[b] = stat == 0 ? (banned || prm.warm_valid[b] == 2 ? 2 : 1) : 0;
  }

  // ---- 6b. differentiable mode: what the adjoint solve of this optimum needs (nrmp_adjoint_kernel) ----------------
  double* arec = prm.adj_save ? prm.adj_save + (size_t)b * nrmp_adj_doubles(T, M) : nullptr;
  const bool adj_ok = arec != nullptr && stat == 0 && have_factor;
  const int oL = 0, oI = (nU * (nU + 3)) >> 1, oF = oI + nU, oP = oF + 3 * FT, oS = oP + 5 * T, oU0 = oS + 3 * T;
  if (arec) {
    __syncwarp();
    if (adj_ok) {
      NB_LL(i, (nU * (nU + 3)) >> 1) arec[oL + i] = H[i];
      if (lane < nU) arec[oI + lane] = invd0;
      if (!SMALL && lane + 32 < nU) arec[oI + lane + 32] = invd1;
      NB_LL(i, 3 * FT) arec[oF + i] = F[i];
      NB_LL(t, T) {
        const bool hasD = TD > 0;
        arec[oP + t] = hasD ? iHDD[t] : 0.0;
        arec[oP + T + t] = hasD ? n0[t] : 0.0;
        arec[oP + 2 * T + t] = hasD ? n1[t] : 0.0;
        arec[oP + 3 * T + t] = (hasD && !dfix) ? cz[oDU + t] * (double)cis[oDU + t] : 0.0;
        arec[oP + 4 * T + t] = (hasD && !dfix) ? cz[oDL + t] * (double)cis[oDL + t] : 0.0;
        arec[oU0 + t] = x[2 * t];
      }
    }
    if (lane == 0) prm.adj_valid[b] = adj_ok ? 1 : 0;
    __syncwarp();
  }

  // ---- 7. outputs: S = s0 + F u, U, D cast to float32 (nrmp.py:145-148) --------------------------
  float* os = prm.out_s + (size_t)b * 3 * T1;
  float* ou = prm.out_u + (size_t)b * 2 * T;
  float* od = prm.out_d + (size_t)b * T;
  const bool keep_nominal = (stat & 6) != 0;  // numeric failure / infeasible: hand back the nominal
  __syncwarp();
  const float init_s = lane < 3 ? ns[lane * T1] : 0.f;  // initial state column (robot.py:234)
  NB_LL(t, T) {
    double sx = s0[t], sy = s0[T + t], sth = s0[2 * T + t];
    for (int i = 0; i < 2 * (t + 1); ++i) {
      sx += F[t * (t + 1) + i] * x[i]; sy += F[FT + t * (t + 1) + i] * x[i]; sth += F[2 * FT + t * (t + 1) + i] * x[i];
    }
    if (keep_nominal) { sx = ns[t + 1]; sy = ns[T1 + t + 1]; sth = ns[2 * T1 + t + 1]; }
    if (adj_ok) { arec[oS + t] = sx; arec[oS + T + t] = sy; arec[oS + 2 * T + t] = sth; }
    // stash (H is dead) so that every read of nom_s is complete before any write (out may alias nom)
    H[3 * t] = sx; H[3 * t + 1] = sy; H[3 * t + 2] = sth;
  }
  NB_LL(i, nU) rdU[i] = keep_nominal ? (double)nu[(i & 1) * T + (i >> 1)] : x[i];
  __syncwarp();
  if (lane < 3) os[lane * T1] = init_s;
  NB_LL(t, T) {
    os[t + 1] = (float)H[3 * t]; os[T1 + t + 1] = (float)H[3 * t + 1]; os[2 * T1 + t + 1] = (float)H[3 * t + 2];
    od[t] = TD > 0 ? (float)Dv[t] : 0.f;
  }
  NB_LL(i, nU) ou[(i & 1) * T + (i >> 1)] = (float)rdU[i];
  if (lane == 0) {
    if (prm.status) prm.status[b] = stat;
    if (prm.iters) prm.iters[b] += 1;
    if (prm.ipm_iters) prm.ipm_iters[b] = it;
  }
  __syncwarp();

  // ---- 8. stop criterion (pan.py:215-243) ----------------------------------------------------------
  if (!prm.defer_stop) nrmp_stop_env<TT, MM>(prm, b, lane);
}

// ---- adjoint of one NRMP solve (differentiable mode; replaces the backward pass of CvxpyLayer, nrmp.py:144) -----------------
// One warp per environment.  With M = P + Ab' W Ab + J' omega J the reduced KKT matrix of the barrier problem at the optimum
// (its U-block Schur complement is the matrix the forward solve factorised last), dx/dtheta = -M^-1 dF/dtheta, hence
//   M z = g_x,   g_x = (F' dL/dS + dL/dU, dL/dD);       dL/dtheta_i = -z' dF/dtheta_i
// with the parameter dependence of the stationarity residual F (gamma_a = q_s ref_s and gamma_b = p_u ref_us included):
//   dF/dq_r   = 4 q_r sum_t F_t[r]' (S_r - ref_r)_{t+1}      (r < 2 for omni)      dF/dp_u = 4 p_u (U0_t - ref_us_t) e_{u0,t}
//   dF/deta   = -e_D        dF/dd_max = -W_Dmax e_D        dF/dd_min = -W_Dmin e_D        dF/dpara_s[r,t+1] = -bk F_t[r]'
// The last one is the gradient that flows on into the previous PAN iteration, whose output S is this solve's `para_s`
// (pan.py:131-142: nom_s is passed on as a tensor; A, B, C, fa, fb are rebuilt from detached values and carry no gradient).
__global__ void __launch_bounds__(128) nrmp_adjoint_kernel(const NrmpAdjParams prm) {
  extern __shared__ __align__(16) double smem_adj[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpc = blockDim.x >> 5;
  const int b = blockIdx.x * wpc + warp;
  if (b >= prm.B) return;
  const int T = prm.T, T1 = T + 1, nU = 2 * T, FT = T * (T + 1);
  const bool hasD = prm.M > 0;
  const int nL = (nU * (nU + 3)) >> 1;
  const int oI = nL, oF = oI + nU, oP = oF + 3 * FT, oS = oP + 5 * T, oU0 = oS + 3 * T;
  double* gs = prm.g_s + (size_t)b * 3 * T1;
  double* gu = prm.g_u + (size_t)b * 2 * T;
  double* gd = prm.g_d + (size_t)b * T;
  if (prm.iters[b] <= prm.k) return;  // this environment had stopped before iteration k: its gradient passes through unchanged
  const bool ok = prm.rec_valid[b] != 0;
  const double* rec = prm.rec + (size_t)b * nrmp_adj_doubles(T, prm.M);
  // per-warp workspace: L (nL) | zU (nU) | qz (3T) | zD (T) | v (T)
  double* w = smem_adj + (size_t)warp * (nL + nU + 5 * T);
  double* L = w; double* zU = L + nL; double* qz = zU + nU; double* zD = qz + 3 * T; double* vv = zD + T;
  auto hrow = [](int i) { return (i * (i + 3)) >> 1; };
  if (!ok) {  // no usable factor (solver status != 0): no gradient through this solve
    for (int i = lane; i < 3 * T1; i += 32) gs[i] = 0.0;
    for (int i = lane; i < 2 * T; i += 32) gu[i] = 0.0;
    for (int i = lane; i < T; i += 32) gd[i] = 0.0;
    return;
  }
  for (int i = lane; i < nL; i += 32) L[i] = rec[i];
  for (int t = lane; t < T; t += 32) vv[t] = hasD ? gd[t] * rec[oP + t] : 0.0;  // g_D / H_DD
  __syncwarp();
  // right-hand side of the U block:  g_U + F' g_S + sum_t F_t[xy]' n_t (g_D / H_DD)_t
  double r0 = 0.0, r1 = 0.0;
  for (int sl = 0; sl < 2; ++sl) {
    const int j = lane + 32 * sl;
    if (j < nU) {
      double acc = gu[(j & 1) * T + (j >> 1)];
      for (int t = j >> 1; t < T; ++t) {
        const int o = t * (t + 1) + j;
        const double fx = rec[oF + o], fy = rec[oF + FT + o], fth = rec[oF + 2 * FT + o];
        acc += fx * (gs[t + 1] + rec[oP + T + t] * vv[t]) + fy * (gs[T1 + t + 1] + rec[oP + 2 * T + t] * vv[t]) + fth * gs[2 * T1 + t + 1];
      }
      if (sl == 0) r0 = acc; else r1 = acc;
    }
  }
  const double invd0 = lane < nU ? rec[oI + lane] : 0.0, invd1 = lane + 32 < nU ? rec[oI + lane + 32] : 0.0;
  for (int k = 0; k < nU; ++k) {  // L y = r
    const double mine = k < 32 ? r0 * invd0 : r1 * invd1;
    const double yk = __shfl_sync(0xffffffffu, mine, k & 31);
    if (lane == (k & 31)) { if (k < 32) r0 = yk; else r1 = yk; }
    if (lane > k && lane < nU) r0 -= L[hrow(lane) + k] * yk;
    if (lane + 32 > k && lane + 32 < nU) r1 -= L[hrow(lane + 32) + k] * yk;
  }
  for (int k = nU - 1; k >= 0; --k) {  // L' z = y
    const double mine = k < 32 ? r0 * invd0 : r1 * invd1;
    const double xk = __shfl_sync(0xffffffffu, mine, k & 31);
    if (lane == (k & 31)) { if (k < 32) r0 = xk; else r1 = xk; }
    if (lane < k) r0 -= L[hrow(k) + lane] * xk;
    if (lane + 32 < k) r1 -= L[hrow(k) + lane + 32] * xk;
  }
  if (lane < nU) zU[lane] = r0;
  if (lane + 32 < nU) zU[lane + 32] = r1;
  __syncwarp();
  for (int t = lane; t < T; t += 32) {  // qz_r[t] = F_t[r] z_U,  z_D
    double a0 = 0, a1 = 0, a2 = 0;
    for (int i = 0; i < 2 * (t + 1); ++i) {
      const int o = t * (t + 1) + i;
      a0 += rec[oF + o] * zU[i]; a1 += rec[oF + FT + o] * zU[i]; a2 += rec[oF + 2 * FT + o] * zU[i];
    }
    qz[t] = a0; qz[T + t] = a1; qz[2 * T + t] = a2;
    zD[t] = hasD ? (gd[t] + rec[oP + T + t] * a0 + rec[oP + 2 * T + t] * a1) * rec[oP + t] : 0.0;
  }
  __syncwarp();
  // parameter gradients
  const float* rs = prm.ref_s + (size_t)b * 3 * T1;
  const float* rus = prm.ref_us + (size_t)b * T;
  const int rows_s = prm.kin == 2 ? 2 : 3;
  double dq[3] = {0, 0, 0}, dpu = 0, deta = 0, ddmax = 0, ddmin = 0;
  for (int t = lane; t < T; t += 32) {
    for (int r = 0; r < rows_s; ++r) dq[r] += -4.0 * (double)prm.q[r] * qz[r * T + t] * (rec[oS + r * T + t] - (double)rs[r * T1 + t + 1]);
    dpu += -4.0 * (double)prm.p_u * zU[2 * t] * (rec[oU0 + t] - (double)rus[t]);
    deta += zD[t];
    ddmax += zD[t] * rec[oP + 3 * T + t];
    ddmin += zD[t] * rec[oP + 4 * T + t];
  }
  for (int r = 0; r < 3; ++r) dq[r] = warp_sum(dq[r]);
  dpu = warp_sum(dpu); deta = warp_sum(deta); ddmax = warp_sum(ddmax); ddmin = warp_sum(ddmin);
  if (lane == 0) {
    double* g = prm.grad_theta + (size_t)b * 7;
    g[0] += dq[0]; g[1] += dq[1]; g[2] += dq[2]; g[3] += dpu; g[4] += deta; g[5] += ddmax;
    g[6] += prm.d_min > 0.f ? ddmin : 0.0;  // the program uses max(d_min, 0) (nonneg Variable, nrmp.py:264-266)
  }
  __syncwarp();
  // what flows on into the previous iteration: dL/dpara_s[r, t+1] = bk F_t[r] z_U; nothing through U, D or the initial column
  for (int i = lane; i < 3 * T1; i += 32) {
    const int r = i / T1, c = i - r * T1;
    gs[i] = c == 0 ? 0.0 : prm.bk * qz[r * T + c - 1];
  }
  for (int i = lane; i < 2 * T; i += 32) gu[i] = 0.0;
  for (int i = lane; i < T; i += 32) gd[i] = 0.0;
}

// Kernel: persistent warps.  Every warp owns one workspace in shared memory and pulls environments from a global counter
// (prm.work_counter, zeroed by the launcher) until the batch is exhausted: solves take 8..25 interior point iterations, so
// a static env -> warp map leaves the fast warps of a wave idle (and a CTA slot is only re-used when BOTH its warps are done).
// work_counter == nullptr: one environment per warp (b = blockIdx.x * warps + warp), the grid covers the batch.
template <int HPL, bool SMALL, int TT, int MM>
#ifndef NB_NRMP_WPC
#define NB_NRMP_WPC 3  // warps per CTA of the (10, 10) specialisation: 3 x 5 CTAs = 15 warps per SM (NB_NRMP_WPC is a tuning knob: 2 x 7 and 1 x 14 are the alternatives to time with bench.py)
#endif
__global__ void __launch_bounds__((TT == 10 && MM == 10) ? 32 * NB_NRMP_WPC : 64, (TT == 10 && MM == 10) ? (NB_NRMP_WPC == 3 ? 5 : (NB_NRMP_WPC == 1 ? 14 : 7)) : (HPL <= 4 ? 6 : 4))
    nrmp_kernel(const NrmpParams prm, int warps_per_cta, int warp_doubles_rt) {
  extern __shared__ __align__(16) double smem_d[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int T = TT > 0 ? TT : prm.T, M = TT > 0 ? MM : prm.M;
  const int warp_doubles = TT > 0 ? (int)nrmp_warp_doubles(TT, MM) : warp_doubles_rt;
  const int nU = 2 * T, nP = nU * (nU + 1) / 2;
  (void)M;
  // pair table (i << 8 | j) of the lower triangle, shared by the CTA
  unsigned short* ptab = reinterpret_cast<unsigned short*>(smem_d + (size_t)warps_per_cta * warp_doubles);
  for (int p = threadIdx.x; p < nP; p += blockDim.x) {
    int i = (int)((sqrtf(8.0f * p + 1.0f) - 1.0f) * 0.5f);
    while (i * (i + 1) / 2 > p) --i;
    while ((i + 1) * (i + 2) / 2 <= p) ++i;
    ptab[p] = (unsigned short)((i << 8) | (p - i * (i + 1) / 2));
  }
  __syncthreads();
  double* wsp = smem_d + (size_t)warp * warp_doubles;
  // one call site (one inlined copy of the solve: the code is ~60 KB): without a counter the loop body runs once for the warp's own env
  bool first = true;
#pragma unroll 1
  for (;;) {
    int b = 0;
    if (prm.work_counter != nullptr) {
      if (lane == 0) b = atomicAdd(prm.work_counter, 1);
      b = __shfl_sync(0xffffffffu, b, 0);
    } else {
      if (!first) break;
      first = false;
      b = blockIdx.x * warps_per_cta + warp;
    }
    if (b >= prm.B) break;
    if (prm.active && prm.active[b] == 0) continue;
    nrmp_solve_env<HPL, SMALL, TT, MM>(prm, b, wsp, ptab, lane);
    __syncwarp();
  }
}

// the deferred section 8: one warp per environment, the same arithmetic in the same order as inside the solve
__global__ void __launch_bounds__(128) nrmp_stop_kernel(const NrmpParams prm) {
  const int lane = threadIdx.x & 31, b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= prm.B) return;
  if (prm.active && prm.active[b] == 0) return;
  nrmp_stop_env<0, 0>(prm, b, lane);
}

#undef NB_PHASE
#undef NB_LW
#undef NB_LL
}  // namespace nb
