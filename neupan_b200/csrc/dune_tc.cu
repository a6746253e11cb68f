// Translation unit of the warpgroup (wgmma) DUNE kernels: host-side operand image + launchers.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "host_common.h"
#include "dune_tc_kernel.cuh"
#include "dune_screen_kernel.cuh"
#include "dune_screen_mma_kernel.cuh"

namespace nb {

static inline void split_half_tc(float v, uint16_t& hi, uint16_t& lo) {
  const __half h = __float2half_rn(v);
  const __half l = __float2half_rn(v - __half2float(h));
  memcpy(&hi, &h, 2);
  memcpy(&lo, &l, 2);
}

// packed checkpoint (WeightLayout order, E outputs) -> TcImage bytes (canonical K-major / no-swizzle wgmma layout)
// returns flags: bit 0 = every tanh argument of the network is bounded by 30 in exp2 units (|LN(x)_j| <= sqrt(32)), which
// allows the kernel's shared-reciprocal tanh (ln_tanh_split<true>)
// screen = true: the image of the screening network (dune_screen_kernel.cuh): the same layout, but tanh is NOT folded into the
// following layer (the screen kernel applies MUFU.TANH itself) and the LayerNorm gain / offset are the checkpoint's plain values;
// only the hi halves of the weights are used.
int build_tc_image(const float* w, int E, std::vector<unsigned char>& out, bool screen) {
  using L = WeightLayout;
  using I = TcImage;
  out.assign(I::kBytes, 0);
  auto put = [&](size_t off, uint16_t v) { memcpy(out.data() + off, &v, 2); };
  // element (n, k) of a K-major operand with `lbo` bytes between the two 8-half K groups and `kstep` bytes per 16 of K
  auto at = [](int n, int k, int lbo, int kstep) { return (size_t)(k / 16) * kstep + ((k % 16) / 8) * lbo + (n / 8) * 128 + (n % 8) * 16 + (k % 8) * 2; };
  float* fl = reinterpret_cast<float*>(out.data() + I::kFloatOff);
  // the five dense layers: MLP.3, .5, .8, .10 and the head MLP.13 (E rows, zero padded to N = 32).
  // Layers fed by a tanh (MLP.3, MLP.8, MLP.13) receive r = 1/(exp(2y)+1) instead of tanh(y) = 1 - 2r:
  //   W tanh + b = (b + rowsum(W)) + (-2 W) r
  const int dense_w[5] = {L::W3, L::W5, L::W8, L::W10, L::W13}, dense_b[5] = {L::B3, L::B5, L::B8, L::B10, L::b13(E)};
  const int rows[5] = {32, 32, 32, 32, E};
  const bool after_tanh[5] = {!screen, false, !screen, false, !screen};
  // Layers that feed a LayerNorm (MLP.0 -> LN1, MLP.5 -> LN6, MLP.10 -> LN11) are CENTRED here: LN subtracts the mean over
  // the 32 outputs, which is linear, so W - colmean(W) and b - mean(b) deliver mean-free pre-activations for free.
  const bool before_ln[5] = {false, true, false, true, false};
  for (int l = 0; l < 5; ++l) {
    const size_t base = (size_t)l * I::kLayerStride;
    std::vector<double> W(32 * 32, 0.0), bv(32, 0.0);
    for (int n = 0; n < rows[l]; ++n) {
      double rowsum = 0.0;
      for (int k = 0; k < 32; ++k) {
        const double wv = (double)w[dense_w[l] + n * 32 + k];
        rowsum += wv;
        W[n * 32 + k] = after_tanh[l] ? -2.0 * wv : wv;
      }
      bv[n] = (double)w[dense_b[l] + n] + (after_tanh[l] ? rowsum : 0.0);
    }
    if (before_ln[l]) {
      for (int k = 0; k < 32; ++k) {
        double m = 0.0;
        for (int n = 0; n < 32; ++n) m += W[n * 32 + k];
        for (int n = 0; n < 32; ++n) W[n * 32 + k] -= m / 32;
      }
      double m = 0.0;
      for (int n = 0; n < 32; ++n) m += bv[n];
      for (int n = 0; n < 32; ++n) bv[n] -= m / 32;
    }
    for (int n = 0; n < 32; ++n) {
      for (int k = 0; k < 32; ++k) {
        uint16_t hi, lo;
        split_half_tc((float)W[n * 32 + k], hi, lo);
        put(base + at(n, k, 512, 1024), hi);
        put(base + 2048 + at(n, k, 512, 1024), lo);
      }
      fl[I::BH + 32 * l + n] = (float)bv[n];
    }
  }
  for (int m = 0; m < 128; ++m)  // ONES(m, 0..2) = 1.0h, K-major with 2048 B between the two 8-wide K groups
    for (int k = 0; k < 3; ++k) put(I::kOnesOff + (size_t)(m / 8) * 128 + (m % 8) * 16 + k * 2, 0x3C00);
  for (int l = 0; l < 5; ++l)    // BIASB[l](n, 0..2) = three fp16 pieces of the (folded) bias
    for (int n = 0; n < 32; ++n) {
      float rest = fl[I::BH + 32 * l + n];
      for (int k = 0; k < 3; ++k) {
        const __half h = __float2half_rn(rest);
        rest -= __half2float(h);
        uint16_t bits;
        memcpy(&bits, &h, 2);
        put(I::kBiasBOff + (size_t)l * 1024 + at(n, k, 512, 1024), bits);
      }
    }
  {  // layer 0 (2 -> 32), centred for LN1; both layouts (row-major for the first kernel, columns for the packed one)
    double mx = 0.0, my = 0.0, mb = 0.0;
    for (int j = 0; j < 32; ++j) { mx += w[L::W0 + 2 * j]; my += w[L::W0 + 2 * j + 1]; mb += w[L::B0 + j]; }
    for (int j = 0; j < 32; ++j) {
      fl[I::W0X + j] = (float)((double)w[L::W0 + 2 * j] - mx / 32);
      fl[I::W0Y + j] = (float)((double)w[L::W0 + 2 * j + 1] - my / 32);
      fl[I::W0 + 2 * j] = fl[I::W0X + j];
      fl[I::W0 + 2 * j + 1] = fl[I::W0Y + j];
      fl[I::B0 + j] = (float)((double)w[L::B0 + j] - mb / 32);
    }
  }
  const int g_src[3] = {L::G1, L::G6, L::G11}, b_src[3] = {L::BE1, L::BE6, L::BE11};
  const int g_dst[3] = {I::G1, I::G6, I::G11}, b_dst[3] = {I::BE1, I::BE6, I::BE11};
  for (int q = 0; q < 3; ++q)
    for (int i = 0; i < 32; ++i) {  // pre-multiplied by 2*log2(e): tanh(y) = 1 - 2/(exp2(2*log2(e)*y) + 1)
      const double sc = screen ? 1.0 : 2.8853900817779268;
      fl[g_dst[q] + i] = (float)((double)w[g_src[q] + i] * sc);
      fl[b_dst[q] + i] = (float)((double)w[b_src[q] + i] * sc);
    }
  double amax = 0.0;
  for (int q = 0; q < 3; ++q)
    for (int i = 0; i < 32; ++i) {
      const double a = std::fabs((double)fl[g_dst[q] + i]) * 5.6568542494923806 + std::fabs((double)fl[b_dst[q] + i]);  // sqrt(32)
      if (!(a <= amax)) amax = a;  // NaN-propagating max
    }
  return amax <= 30.0 ? 1 : 0;
}

// persistent grid: as many CTAs as fit on every SM, at most `work` (0: the kernel does not fit at all)
template <typename K>
static cudaError_t resident_grid(K kern, int threads, size_t smem, int sm_count, int work, int& grid) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  int per_sm = 0;
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem);
  grid = sm_count * (per_sm < 1 ? 1 : per_sm);
  if (grid > work) grid = work;
  return e;
}

// screen = false: dune_tcp_kernel on every point (NB_OPT_DUNE_KERNEL = 2); true: the screening pipeline (4).  The shared-reciprocal
// tanh is taken wherever image_flags allows it, in the refine and the exact kernel alike, so both pipelines compute the same bits.
// Counts its launches (3 with screening, 1 without) once all of them are enqueued.
int launch_dune_tc(const DuneParams& prm_in, const unsigned char* d_image, const unsigned char* d_screen_image, int image_flags, bool screen, int sm_count,
                   int max_smem_optin, cudaStream_t st) {
  DuneParams prm = prm_in;
  const bool fast = (image_flags & 1) != 0;
  if (screen) {
    // screening: (1) interval pass over all points, (2) exact evaluation of the candidates, (3) the exact kernel for the items the
    // screen could not narrow down to 32 candidates (below, with only_flagged)
    if (!d_screen_image || !prm.cand_idx || !prm.cand_cnt || !prm.cand_dt || !prm.cand_rad || !prm.screen_stats || !prm.flag_list || !prm.flag_count || !prm.refine_list)
      return fail(NB_ERR_INVALID, "screening buffers are not allocated");
    const int items_ = prm.B * (prm.T + 1);
    const size_t smem_s = dune_screen_smem_bytes(prm.N, prm.M);
    if ((long long)smem_s > max_smem_optin)
      return fail(NB_ERR_CAPACITY, "N=%d needs %zu B of shared memory (limit %d)", prm.N, smem_s, max_smem_optin);
    const size_t smem_r = TcImage::kBytes + 2 * (size_t)tc::kTileBytes;
    const int screen_mma = prm.screen_mma;
    cudaError_t e = cudaMemsetAsync(prm.flag_count, 0, 3 * sizeof(int32_t), st);
    const bool warp_items = prm.N <= 32 * kWarpTiles;  // one warp per item, CTAs persistent over environments
    const size_t smem_m = warp_items ? dune_screen_warp_smem_bytes(prm.N, prm.T) : dune_screen_mma_smem_bytes(prm.N, prm.M);
    int grid = 0;
    if (screen_mma && prm.N <= 1024 && (long long)smem_m <= max_smem_optin) {  // larger clouds: the warpgroup screen kernel (key arrays in shared memory)
      auto go = [&](auto kern, int threads, int work, auto... args) {
        if (e == cudaSuccess) e = resident_grid(kern, threads, smem_m, sm_count, work, grid);
        if (e == cudaSuccess) {
          static int cap = -1;  // NB_SCREEN_CTA_CAP (developer switch): fewer CTAs per SM, to leave room for a kernel of another stream (NB_OPT_OVERLAP)
          if (cap < 0) {
            const char* v = getenv("NB_SCREEN_CTA_CAP");
            cap = v ? atoi(v) : 0;
          }
          if (cap > 0 && grid > sm_count * cap) grid = sm_count * cap;
          kern<<<grid, threads, smem_m, st>>>(prm, d_screen_image, args...);
          e = cudaGetLastError();
        }
      };
      if (warp_items) {
        // one CTA per environment leaves SMs idle when the batch is smaller than the resident grid: split the items over more
        int resident = 0;
        if (e == cudaSuccess) e = resident_grid(dune_screen_warp_kernel, 32 * kScreenWarps, smem_m, sm_count, 1 << 30, resident);
        const int groups = (prm.T + 1 + kScreenWarps - 1) / kScreenWarps;
        int parts = resident / (prm.B > 0 ? prm.B : 1);
        parts = parts < 1 ? 1 : (parts > groups ? groups : parts);
        go(dune_screen_warp_kernel, 32 * kScreenWarps, prm.B * parts, parts);
      } else {
        go(dune_screen_mma_kernel, 128, items_);
      }
    } else {
      if (e == cudaSuccess) e = resident_grid(dune_screen_kernel<0>, 128, smem_s, sm_count, items_, grid);
      if (e == cudaSuccess) {
        dune_screen_kernel<0><<<grid, 128, smem_s, st>>>(prm, d_screen_image);
        e = cudaGetLastError();
      }
    }
    const int groups = (items_ + 7) / 8;  // the number of work units is only known on the device: a persistent grid sized for the worst case
    if (e == cudaSuccess) e = fast ? resident_grid(dune_refine_kernel<true>, 128, smem_r, sm_count, groups, grid)
                                    : resident_grid(dune_refine_kernel<false>, 128, smem_r, sm_count, groups, grid);
    if (e == cudaSuccess) {
      if (fast) dune_refine_kernel<true><<<grid, 128, smem_r, st>>>(prm, d_image);
      else dune_refine_kernel<false><<<grid, 128, smem_r, st>>>(prm, d_image);
      e = cudaGetLastError();
    }
    if (e != cudaSuccess) return fail(NB_ERR_CUDA, "dune screen / refine launch failed: %s", cudaGetErrorString(e));
    prm.only_flagged = 1;
  }
  const size_t smem = dune_tc_smem_bytes(prm.N, prm.geo.E, prm.M);
  if ((long long)smem > max_smem_optin) return fail(NB_ERR_CAPACITY, "N=%d needs %zu B of shared memory (limit %d)", prm.N, smem, max_smem_optin);
  const int items = prm.B * (prm.T + 1);
  auto run = [&](auto kern) -> cudaError_t {
    int grid = 0;
    cudaError_t e = resident_grid(kern, 128, smem, sm_count, items, grid);
    if (e != cudaSuccess) return e;
    kern<<<grid, 128, smem, st>>>(prm, d_image);
    return cudaGetLastError();
  };
  const cudaError_t e = fast ? run(dune_tcp_kernel<true>) : run(dune_tcp_kernel<false>);
  if (e != cudaSuccess) return fail(NB_ERR_CUDA, "dune_tc kernel launch failed: %s", cudaGetErrorString(e));
  launches += screen ? 3 : 1;
  return NB_OK;
}

}  // namespace nb
