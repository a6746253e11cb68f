// Definitions shared by the NRMP kernels (nrmp_kernel.cuh) and the host code that drives them: the launch parameters, the
// shared-memory and record sizes, and the launchers (nrmp.cu).
#pragma once
#include "common.cuh"

namespace nb {
struct NrmpParams {
  const float* nom_s;   // (B,3,T+1) nominal states in
  const float* nom_u;   // (B,2,T)
  const float* ref_s;   // (B,3,T+1)
  const float* ref_us;  // (B,T)
  const float* fa;      // (B,T,M,2) explicit coefficients or nullptr
  const float* fb;      // (B,T,M)
  const float* sel_mu;  // (B,T+1,M,E) DUNE selections (used when fa == nullptr) or nullptr
  const float* sel_lam; // (B,T+1,M,2)
  const float* sel_pts; // (B,T+1,M,2)
  const int32_t* sel_count;  // (B)
  float* out_s;         // (B,3,T+1)  may alias nom_s (each warp reads its env before writing)
  float* out_u;         // (B,2,T)
  float* out_d;         // (B,T)
  int32_t* status;      // (B) or nullptr
  int32_t* iters;       // (B) or nullptr: incremented per executed iteration
  int32_t* ipm_iters;   // (B) or nullptr: interior point iterations of this solve (diagnostics)
  int32_t* active;      // (B) or nullptr: envs with 0 are skipped; cleared when the stop test fires
  // PAN.current_nom_values (pan.py:100-105), per env; nullptr disables the stop criterion
  float* prev_s; float* prev_u; float* prev_mu; float* prev_lam; int32_t* prev_count; int32_t* prev_valid;
  // warm start (NB_OPT_NRMP_WARM): per-env float record [x (2T) | D (T) | z of the box/rate/D rows (mb) | z of the hinge rows (T*M)]
  // of the last converged solve; warm_valid[b] != 0 marks it usable.  nullptr = always cold.
  float* warm; int32_t* warm_valid;
  int warm_check_it; double warm_check_gap;  // a warm start whose gap is still above warm_check_gap at iteration warm_check_it restarts cold
  int* work_counter;  // dynamic env -> warp assignment (see nrmp_kernel), or nullptr
  int defer_stop;     // 1 = the solve kernel leaves the stop criterion / PAN.current_nom_values update (section 8) to nrmp_stop_kernel
  // differentiable mode (LON, SURVEY 8f row 3): per-env record of this solve for nrmp_adjoint_kernel, nrmp_adj_doubles(T, M)
  // doubles each, and a validity flag; nullptr = inference
  double* adj_save; int32_t* adj_valid;
  int B, T, M, E, kin;
  int max_ipm_iter;
  double gap_tol;  // mean complementarity at termination (1e-12; the one-row hinge form has no degenerate pairs that would dominate the mean, so the same accuracy in u needs a smaller number than the 1e-10 of the two-row form)
  float iter_threshold;
  double dt, L;
  float q[3], p_u, eta, d_max, d_min;
  double ro, bk;
  double speed[2], acce[2];  // speed_bound, acce_bound = max_acce*dt (robot.py:68-69)
  float h[kMaxEdges];
};


// per-warp shared memory, in doubles
__host__ __device__ inline size_t nrmp_scratch_doubles(int T, int M) {
  size_t sc = 2 * (size_t)T * (T + 1);  // Gx,Gy (packed like F); also holds per-hinge scratch (T*M) and the setup-only linearisation (12 T)
  if (sc < (size_t)T * M) sc = (size_t)T * M;
  if (sc < 12 * (size_t)T) sc = 12 * (size_t)T;
  return sc;
}
__host__ __device__ inline size_t nrmp_warp_doubles(int T, int M) {
  const int nU = 2 * T, nR = nU - 2, TD = M > 0 ? T : 0, TM = T * M;
  const int mb = 2 * nU + 2 * nR + 2 * TD;
  size_t n = 0;
  n += 3 * (size_t)T * (T + 1);    // F, packed: row t keeps only its 2(t+1) structurally non-zero columns at offset t(t+1)
  n += 3 * (size_t)T;              // s0
  n += (size_t)nU * (nU + 1) / 2;  // Hc
  n += (size_t)nU * (nU + 3) / 2;  // H / Cholesky factor: lower triangle, row i at i(i+3)/2 (one pad element per row)
  n += nrmp_scratch_doubles(T, M);
  n += 4 * (size_t)nU;             // cv, x, rdU, dU
  n += 14 * (size_t)T;             // per-step scalars
  n += 4 * (size_t)mb;             // s, z, ds, dz of the box / rate / D rows
  n += ((size_t)mb + 1) / 2;       // is (float)
  n += (size_t)TM;                 // fax, fay (float)
  return n + 1;
}
__host__ __device__ inline size_t nrmp_cta_extra_bytes(int T) {  // pair table (uint16) shared by the CTA's warps
  const int nU = 2 * T;
  return (((size_t)nU * (nU + 1) / 2) * 2 + 15) / 16 * 16;
}

// adjoint record of one solve: [L (nU(nU+3)/2) | 1/diag(L) (nU) | F x,y,theta (3 T(T+1)) | 1/H_DD, n0, n1, W_Dmax, W_Dmin (5T) |
// S rows x,y,theta at t = 1..T (3T) | U0 (T)]
__host__ __device__ inline size_t nrmp_adj_doubles(int T, int M) {
  const size_t nU = 2 * (size_t)T;
  (void)M;
  return nU * (nU + 3) / 2 + nU + 3 * (size_t)T * (T + 1) + 9 * (size_t)T;
}

__host__ __device__ inline size_t nrmp_warm_floats(int T, int M) {
  const int nU = 2 * T, nR = nU - 2, TD = M > 0 ? T : 0;
  return (size_t)nU + TD + (2 * nU + 2 * nR + 2 * TD) + (size_t)T * M;
}

// adjoint of one NRMP solve (nrmp_adjoint_kernel, differentiable mode)
struct NrmpAdjParams {
  const double* rec;         // (B, nrmp_adj_doubles)
  const int32_t* rec_valid;  // (B)
  const int32_t* iters;      // (B) iterations executed by the forward; the record is this iteration's iff iters[b] > k
  int k;
  const float* ref_s;        // (B,3,T+1)
  const float* ref_us;       // (B,T)
  double* g_s;               // (B,3,T+1) upstream dL/dS on entry, dL/dpara_s for the previous iteration on exit
  double* g_u;               // (B,2,T)   upstream dL/dU on entry, zero on exit
  double* g_d;               // (B,T)     upstream dL/dD on entry, zero on exit
  double* grad_theta;        // (B,7) accumulated: q0, q1, q2, p_u, eta, d_max, d_min
  int B, T, M, kin;
  float q[3], p_u, d_min;
  double bk;
};

// What the calling handle lends an NRMP launch.
struct NrmpLaunch {
  int sm_count, max_smem_optin;
  int defer_stop_min;  // smallest batch whose stop criterion runs as nrmp_stop_kernel
  int dynamic;         // persistent warps pulling environments from work_counter (when the batch exceeds one resident grid)
  int* work_counter;   // the counter of the launching stream
};

// nrmp.cu: one PAN iteration's solves of prm.B environments.  Picks the nrmp_kernel instantiation for (prm.T, prm.M), sets
// prm.defer_stop and prm.work_counter, and launches nrmp_stop_kernel after the solve when the stop criterion is deferred.
int launch_nrmp(NrmpParams prm, const NrmpLaunch& how, cudaStream_t st);

// nrmp.cu: the backward pass of the last forward.  grad_s, grad_u, grad_d (float, nullptr = zero) go into a.g_s, a.g_u, a.g_d, one
// nrmp_adjoint_kernel per PAN iteration runs in reverse over iterations K-1 .. 0 (iteration k's records start at environment
// k * rec_envs of a.rec and a.rec_valid), and the accumulated a.grad_theta comes out as float in grad_theta (a.B x 7).
int launch_nrmp_backward(NrmpAdjParams a, int K, int rec_envs, const float* grad_s, const float* grad_u, const float* grad_d,
                         float* grad_theta, cudaStream_t st);

}  // namespace nb
