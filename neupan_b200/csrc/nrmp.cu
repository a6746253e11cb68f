// Translation unit of the NRMP kernels (nrmp_kernel.cuh) and every launch of them: which instantiation a (T, M) runs, the launch
// shape, the persistent grid, the deferred stop criterion and the backward pass.  NB_NRMP_* -D flags reach the kernels and their
// launcher here alike.
#include <cstdlib>

#include "host_common.h"
#include "nrmp_kernel.cuh"

namespace nb {

namespace {
__global__ void adj_load_kernel(int n_s, int n_u, int n_d, int n_t, const float* gs, const float* gu, const float* gd, double* ds, double* du, double* dd,
                                double* dtheta) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_s) ds[i] = gs ? (double)gs[i] : 0.0;
  if (i < n_u) du[i] = gu ? (double)gu[i] : 0.0;
  if (i < n_d) dd[i] = gd ? (double)gd[i] : 0.0;
  if (i < n_t) dtheta[i] = 0.0;
}
__global__ void adj_store_kernel(int n, const double* dtheta, float* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (float)dtheta[i];
}
}  // namespace

int launch_nrmp(NrmpParams prm, const NrmpLaunch& how, cudaStream_t st) {
  // large batches: the stop criterion's ~1300 dependent global reads per environment leave the solve kernel (where each warp waits for
  // them alone) for a kernel of its own; small batches keep it inside (one launch less per PAN iteration matters more there)
  prm.defer_stop = (prm.prev_valid != nullptr && prm.B >= how.defer_stop_min) ? 1 : 0;
  const size_t wd = nrmp_warp_doubles(prm.T, prm.M);
  const size_t extra = nrmp_cta_extra_bytes(prm.T);
  const int TM = prm.T * prm.M;
  if (TM > 256) return fail(NB_ERR_CAPACITY, "receding*nrmp_max_num = %d exceeds 256", TM);
  int warps = (int)(((size_t)how.max_smem_optin - extra) / (wd * sizeof(double)));
  if (warps < 1) return fail(NB_ERR_CAPACITY, "T=%d, M=%d need %zu B of shared memory per environment", prm.T, prm.M, wd * 8);
  // small CTAs (<= 2 warps): many of them fit per SM and each warp retires independently
  if (warps > 2) warps = 2;
  if (prm.T == 10 && prm.M == 10) warps = NB_NRMP_WPC;
  const size_t smem = (size_t)warps * wd * sizeof(double) + extra;
  int grid = (prm.B + warps - 1) / warps;
  auto go = [&](auto kern) -> int {
    NB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, how.max_smem_optin));
    if (how.dynamic && how.work_counter) {
      // persistent warps: as many CTAs as are resident at once; they pull environments from a counter until the batch is done
      int per_sm = 0;
      NB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, warps * 32, smem));
      static int cap = -1;  // NB_NRMP_CTA_CAP (developer switch): fewer resident CTAs per SM, to share the SMs with a kernel of another stream
      if (cap < 0) {
        const char* v = getenv("NB_NRMP_CTA_CAP");
        cap = v ? atoi(v) : 0;
      }
      if (cap > 0 && cap < per_sm) per_sm = cap;
      const int resident = (per_sm > 0 ? per_sm : 1) * how.sm_count;
      if (grid > resident) {
        grid = resident;
        prm.work_counter = how.work_counter;
        NB_CUDA(cudaMemsetAsync(prm.work_counter, 0, sizeof(int), st));
      }
    }
    kern<<<grid, warps * 32, smem, st>>>(prm, warps, (int)wd);
    ++launches;
    if (prm.defer_stop) {  // section 8 (stop criterion, PAN.current_nom_values) as a bandwidth kernel over the batch
      nrmp_stop_kernel<<<(prm.B + 3) / 4, 128, 0, st>>>(prm);
      ++launches;
    }
    NB_CUDA(cudaGetLastError());
    return NB_OK;
  };
  const int hpl = (TM + 31) / 32;
  // specialisations with compile-time (T, M) for the reference's shipped configurations
  if (prm.T == 10 && prm.M == 10) return go(nrmp_kernel<4, true, 10, 10>);
  if (prm.T == 15 && prm.M == 10) return go(nrmp_kernel<5, true, 15, 10>);
  if (prm.T <= 16) {  // 2T <= 32: one row of the reduced system per lane
    if (hpl <= 1) return go(nrmp_kernel<1, true, 0, 0>);
    if (hpl <= 2) return go(nrmp_kernel<2, true, 0, 0>);
    if (hpl <= 4) return go(nrmp_kernel<4, true, 0, 0>);
    if (hpl <= 5) return go(nrmp_kernel<5, true, 0, 0>);
    return go(nrmp_kernel<8, true, 0, 0>);
  }
  if (hpl <= 4) return go(nrmp_kernel<4, false, 0, 0>);
  return go(nrmp_kernel<8, false, 0, 0>);
}

int launch_nrmp_backward(NrmpAdjParams a, int K, int rec_envs, const float* grad_s, const float* grad_u, const float* grad_d,
                         float* grad_theta, cudaStream_t st) {
  const int T = a.T, T1 = T + 1, nU = 2 * T;
  const int n_s = a.B * 3 * T1, n_u = a.B * 2 * T, n_d = a.B * T, n_t = a.B * 7;
  const int tb = 256, gb = (n_s + tb - 1) / tb;
  adj_load_kernel<<<gb, tb, 0, st>>>(n_s, n_u, n_d, n_t, grad_s, grad_u, grad_d, a.g_s, a.g_u, a.g_d, a.grad_theta);
  ++launches;
  const int wpc = 4;
  const size_t smem = (size_t)wpc * (((size_t)nU * (nU + 3)) / 2 + nU + 5 * T) * sizeof(double);
  if (smem > 48 * 1024) NB_CUDA(cudaFuncSetAttribute(nrmp_adjoint_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const double* rec = a.rec;
  const int32_t* rec_valid = a.rec_valid;
  for (int k = K - 1; k >= 0; --k) {  // reverse over the PAN iterations: the gradient w.r.t. para_s chains into the previous solve
    a.k = k;
    a.rec = rec + (size_t)k * rec_envs * nrmp_adj_doubles(T, a.M);
    a.rec_valid = rec_valid + (size_t)k * rec_envs;
    nrmp_adjoint_kernel<<<(a.B + wpc - 1) / wpc, wpc * 32, smem, st>>>(a);
    ++launches;
  }
  adj_store_kernel<<<(n_t + tb - 1) / tb, tb, 0, st>>>(n_t, a.grad_theta, grad_theta);
  ++launches;
  NB_CUDA(cudaGetLastError());
  return NB_OK;
}

}  // namespace nb

#if NB_NRMP_PHASES
// timing builds only (NB_NRMP_PHASES, tools/nrmp_bench.py --phases): copies the 8 phase counters of nrmp_kernel.cuh to `out` (host),
// then zeroes them when `reset` is set.  Not part of the public header.
extern "C" int nb_nrmp_read_phases(unsigned long long* out, int reset) {
  if (cudaDeviceSynchronize() != cudaSuccess) return NB_ERR_CUDA;
  if (out && cudaMemcpyFromSymbol(out, nb::nb_nrmp_phase_cycles, sizeof(nb::nb_nrmp_phase_cycles)) != cudaSuccess) return NB_ERR_CUDA;
  if (reset) {
    const unsigned long long zero[8] = {};
    if (cudaMemcpyToSymbol(nb::nb_nrmp_phase_cycles, zero, sizeof(zero)) != cudaSuccess) return NB_ERR_CUDA;
  }
  return NB_OK;
}
#endif
