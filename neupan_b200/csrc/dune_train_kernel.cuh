// DUNE training on the device (SURVEY 8f row 4): the reference's DUNETrain (neupan/blocks/dune_train.py:60-384) as two kernels.
//
//  dune_label_kernel   generate_data_set / prob_solve (:100-140): the label of a sampled point p is the solution of the cone program
//                      (10)  max mu'(G p - h)  s.t. |G' mu| <= 1, mu >= 0  -- the dual of the distance from p to the robot polygon --
//                      which the reference obtains from cvxpy/ECOS, one solve per point (100,000 by default).  Closed form (thread per
//                      point, FP64): closest boundary point x*; x* inside edge e -> mu_e = 1/|G_e|; x* a vertex of edges e, f ->
//                      (mu_e, mu_f) >= 0 with G_e' mu_e + G_f' mu_f = (p - x*)/|p - x*|; p inside -> 0.  (oracle/dune_label.py carries
//                      the optimality certificate.)
//  dune_train_epoch_kernel   train_one_epoch (:281-333) for one pass over the data: per batch of <= 256 points the forward of
//                      ObsPointNet, the four-term loss  MSE(mu) + MSE(distance) + MSE(fa) + MSE(fb)  with the batch's random rotation R
//                      (:335-362), the backward pass and torch.optim.Adam's update (lr, betas (0.9, 0.999), eps 1e-8, weight_decay 1e-4 as
//                      L2 on the gradient, :72), all in FP32 like the reference.
//
// Shape of the work: 4,644 parameters, 256 points per optimiser step, and the steps are strictly sequential (every batch sees the
// weights the previous one produced): 20 MFLOP per step.  That is a latency problem, not a throughput problem -- tensor cores
// (128-row tiles, fp16 operands) would add split / operand-tile traffic to a step that is bound by its ~20 block barriers -- so ONE persistent
// CTA keeps the weights in shared memory for the whole epoch and runs thread-per-point FP32 forward/backward passes; the weight
// gradients  dW = delta' a  are small GEMMs over the batch done cooperatively from shared memory (each thread owns four entries per
// layer and, afterwards, the Adam update of exactly those entries).  Pre-activations are recomputed in the backward pass instead of
// stored (layer inputs only: 5 x 32 floats per point), which is what lets a 256-point batch fit in 227 KB.
#pragma once
#include "common.cuh"

namespace nb {

struct DuneLabelParams {
  int n, E;
  float G[kMaxEdges][2];
  float h[kMaxEdges];
  const double* points;  // (n,2) float64 samples (np.random.uniform)
  float* points_f32;     // (n,2) network inputs (np_to_tensor)
  float* mu;             // (n,E)
  float* dist;           // (n)
};

__global__ void dune_label_kernel(const DuneLabelParams prm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= prm.n) return;
  const int E = prm.E;
  const double px = prm.points[2 * i], py = prm.points[2 * i + 1];
  double Gx[kMaxEdges], Gy[kMaxEdges], hh[kMaxEdges], vx[kMaxEdges], vy[kMaxEdges], r[kMaxEdges];
  bool inside = true;
  for (int e = 0; e < E; ++e) {
    Gx[e] = (double)prm.G[e][0]; Gy[e] = (double)prm.G[e][1]; hh[e] = (double)prm.h[e];
    r[e] = Gx[e] * px + Gy[e] * py - hh[e];
    inside = inside && r[e] <= 0.0;
  }
  for (int e = 0; e < E; ++e) {  // vertex e = intersection of rows e and e+1 (cyclic order of gen_inequal_from_vertex)
    const int f = (e + 1) % E;
    const double det = Gx[e] * Gy[f] - Gy[e] * Gx[f];
    vx[e] = (hh[e] * Gy[f] - Gy[e] * hh[f]) / det;
    vy[e] = (Gx[e] * hh[f] - hh[e] * Gx[f]) / det;
  }
  double mu[kMaxEdges];
  for (int e = 0; e < E; ++e) mu[e] = 0.0;
  double value = 0.0;
  if (!inside) {
    double best = 1e300, bt = 0.0, bx = 0.0, by = 0.0;
    int be = 0;
    for (int e = 0; e < E; ++e) {  // row e runs from vertex e-1 to vertex e
      const int a = (e + E - 1) % E;
      const double dx = vx[e] - vx[a], dy = vy[e] - vy[a];
      double t = ((px - vx[a]) * dx + (py - vy[a]) * dy) / (dx * dx + dy * dy);
      t = t < 0.0 ? 0.0 : (t > 1.0 ? 1.0 : t);
      const double xx = vx[a] + t * dx, xy = vy[a] + t * dy;
      const double d = sqrt((px - xx) * (px - xx) + (py - xy) * (py - xy));
      if (d < best) { best = d; be = e; bt = t; bx = xx; by = xy; }
    }
    if (bt > 0.0 && bt < 1.0) {
      mu[be] = 1.0 / sqrt(Gx[be] * Gx[be] + Gy[be] * Gy[be]);
    } else {
      const int f = bt == 0.0 ? (be + E - 1) % E : (be + 1) % E;
      const double nx = (px - bx) / best, ny = (py - by) / best;
      // [G_e' G_f'] (m_e, m_f)' = n
      const double det = Gx[be] * Gy[f] - Gx[f] * Gy[be];
      const double me = (nx * Gy[f] - Gx[f] * ny) / det, mf = (Gx[be] * ny - nx * Gy[be]) / det;
      mu[be] = me > 0.0 ? me : 0.0;
      mu[f] = mf > 0.0 ? mf : 0.0;
    }
    for (int e = 0; e < E; ++e) value += mu[e] * r[e];
  }
  prm.points_f32[2 * i] = (float)px; prm.points_f32[2 * i + 1] = (float)py;
  for (int e = 0; e < E; ++e) prm.mu[(size_t)i * E + e] = (float)mu[e];
  prm.dist[i] = (float)value;
}

// ---- training epoch -------------------------------------------------------------------------------------------------------
struct DuneTrainParams {
  const float* pts;     // (n,2)
  const float* mu;      // (n,E) labels
  const float* dist;    // (n)
  const float* thetas;  // (ceil(n / batch)) rotation angle of every batch (dune_train.py:351-353)
  float* weights;       // packed checkpoint (WeightLayout order), updated in place
  float* adam_m;        // first / second moments, same layout
  float* adam_v;
  double* losses;       // (4) sums over the batches of this pass: mu, distance, fa, fb
  int n, batch, E, validate;
  long long step0;      // optimiser steps taken before this pass (bias correction)
  float lr, beta1, beta2, eps, weight_decay;
  float G[kMaxEdges][2];
  float h[kMaxEdges];
};

constexpr int kTrainThreads = 256;
// per-point vectors live TRANSPOSED in shared memory: feature k of point p at [k * kTrainStride + p].  Point-contiguous rows make a
// thread's own 32 values conflict-free to write / read (lanes = consecutive points) and let the batch GEMMs read four points per
// LDS.128; 260 = 256 + 4 keeps rows 16-byte aligned and spreads the 32 rows over the banks at quarter-warp granularity.
constexpr int kTrainStride = 260;

__host__ __device__ inline size_t dune_train_smem_bytes(int E) {
  const size_t nw = ((size_t)WeightLayout::count(E) + 3) & ~(size_t)3;  // keeps what follows 16-byte aligned
  // weights | a0 (2 rows) | a1..a5 | delta buffer | reduction scratch
  return (nw + 2 * kTrainThreads + 6 * (size_t)32 * kTrainStride + 256) * sizeof(float);
}

namespace train {

// the weights are read from shared memory as float4 (all lanes the same address: one broadcast LDS.128 per four FMAs -- with scalar
// loads the LSU, one warp instruction per clock, was the limit of the whole step)
__device__ __forceinline__ void linear32(const float* __restrict__ W, const float* __restrict__ b, const float (&x)[32], float (&y)[32]) {
#pragma unroll 4
  for (int n = 0; n < 32; ++n) {
    const float4* wr = reinterpret_cast<const float4*>(W + n * 32);
    float acc = b[n], acc2 = 0.f;
#pragma unroll
    for (int k4 = 0; k4 < 8; k4 += 2) {
      const float4 w0 = wr[k4], w1 = wr[k4 + 1];
      acc = fmaf(w0.x, x[4 * k4], acc); acc = fmaf(w0.y, x[4 * k4 + 1], acc); acc = fmaf(w0.z, x[4 * k4 + 2], acc); acc = fmaf(w0.w, x[4 * k4 + 3], acc);
      acc2 = fmaf(w1.x, x[4 * k4 + 4], acc2); acc2 = fmaf(w1.y, x[4 * k4 + 5], acc2); acc2 = fmaf(w1.z, x[4 * k4 + 6], acc2); acc2 = fmaf(w1.w, x[4 * k4 + 7], acc2);
    }
    y[n] = acc + acc2;
  }
}
// x = W' d for a row-major W (32 x 32)
__device__ __forceinline__ void linear32_t(const float* __restrict__ W, const float (&d)[32], float (&x)[32]) {
#pragma unroll
  for (int k = 0; k < 32; ++k) x[k] = 0.f;
#pragma unroll 4
  for (int n = 0; n < 32; ++n) {
    const float dn = d[n];
    const float4* wr = reinterpret_cast<const float4*>(W + n * 32);
#pragma unroll
    for (int k4 = 0; k4 < 8; ++k4) {
      const float4 w = wr[k4];
      x[4 * k4] = fmaf(w.x, dn, x[4 * k4]); x[4 * k4 + 1] = fmaf(w.y, dn, x[4 * k4 + 1]);
      x[4 * k4 + 2] = fmaf(w.z, dn, x[4 * k4 + 2]); x[4 * k4 + 3] = fmaf(w.w, dn, x[4 * k4 + 3]);
    }
  }
}
// LayerNorm (eps 1e-5, biased variance) statistics of h -> xhat (in place), returns rstd
__device__ __forceinline__ float layer_norm32(float (&h)[32]) {
  float m = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) m += h[j];
  m *= 1.0f / 32;
  float v = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) { h[j] -= m; v = fmaf(h[j], h[j], v); }
  const float rstd = rsqrtf(v * (1.0f / 32) + 1e-5f);
#pragma unroll
  for (int j = 0; j < 32; ++j) h[j] *= rstd;
  return rstd;
}
__device__ __forceinline__ void store_row(float* buf, int p, const float (&v)[32]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) buf[j * kTrainStride + p] = v[j];
}
__device__ __forceinline__ void load_row(const float* buf, int p, float (&v)[32]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = buf[j * kTrainStride + p];
}

}  // namespace train

__global__ void __launch_bounds__(kTrainThreads, 1) dune_train_epoch_kernel(const DuneTrainParams prm) {
  extern __shared__ __align__(16) float sm[];
  using L = WeightLayout;
  const int E = prm.E, nw = L::count(E);
  float* W = sm;                                    // packed parameters
  float* a0 = W + ((nw + 3) & ~3);                  // (2, 256): x row, y row
  float* act = a0 + 2 * kTrainThreads;              // a1..a5: 5 x (32 x 260), transposed (see kTrainStride)
  float* dbuf = act + 5 * 32 * kTrainStride;        // 32 x 260: per-point vectors for the batch reductions
  float* red = dbuf + 32 * kTrainStride;            // 32 column sums
  const int tid = threadIdx.x;
  for (int i = tid; i < nw; i += kTrainThreads) W[i] = prm.weights[i];
  __shared__ double loss_acc[4];
  if (tid < 4) loss_acc[tid] = 0.0;
  __syncthreads();

  const int nbatch = (prm.n + prm.batch - 1) / prm.batch;
  // the parameter entries this thread owns: gradient accumulators live in registers, and the owner applies Adam to them.
  //   32x32 layers (W3, W5, W8, W10): entries tid + 256 q, q < 4, i.e. rows n = tid/32 + 8 q, column k = tid % 32
  //   W13 (E x 32): rows n = tid/32 + 8 q < E;  W0 (32 x 2): entries tid < 64;  vectors (biases, LN): tid < 32 (or < E)
  float gW3[4], gW5[4], gW8[4], gW10[4], gW13[1], gW0;
  float gB0, gG1, gBE1, gB3, gB5, gG6, gBE6, gB8, gB10, gG11, gBE11, gB13;
  const int kcol = tid & 31, nrow = tid >> 5;

#pragma unroll 1
  for (int bi = 0; bi < nbatch; ++bi) {
    const int base = bi * prm.batch;
    const int nb = min(prm.batch, prm.n - base);
    const bool live = tid < nb;
    const int pi = base + (live ? tid : 0);
    const float x = prm.pts[2 * pi], y = prm.pts[2 * pi + 1];
    const float th = prm.thetas[bi];
    const float cs = cosf(th), sn = sinf(th);
    // ---------------- forward (thread = point) ----------------
    float v[32], mu_o[kMaxEdges];
    {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = fmaf(W[L::W0 + 2 * j + 1], y, fmaf(W[L::W0 + 2 * j], x, W[L::B0 + j]));
      train::layer_norm32(v);
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = tanhf(fmaf(W[L::G1 + j], v[j], W[L::BE1 + j]));
      a0[tid] = x; a0[kTrainThreads + tid] = y;
      train::store_row(act, tid, v);  // a1
      float u[32];
      train::linear32(W + L::W3, W + L::B3, v, u);
#pragma unroll
      for (int j = 0; j < 32; ++j) u[j] = fmaxf(u[j], 0.f);
      train::store_row(act + 1 * 32 * kTrainStride, tid, u);  // a2
      train::linear32(W + L::W5, W + L::B5, u, v);
      train::layer_norm32(v);
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = tanhf(fmaf(W[L::G6 + j], v[j], W[L::BE6 + j]));
      train::store_row(act + 2 * 32 * kTrainStride, tid, v);  // a3
      train::linear32(W + L::W8, W + L::B8, v, u);
#pragma unroll
      for (int j = 0; j < 32; ++j) u[j] = fmaxf(u[j], 0.f);
      train::store_row(act + 3 * 32 * kTrainStride, tid, u);  // a4
      train::linear32(W + L::W10, W + L::B10, u, v);
      train::layer_norm32(v);
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = tanhf(fmaf(W[L::G11 + j], v[j], W[L::BE11 + j]));
      train::store_row(act + 4 * 32 * kTrainStride, tid, v);  // a5
#pragma unroll
      for (int e = 0; e < kMaxEdges; ++e) {
        mu_o[e] = 0.f;
        if (e < E) {
          float acc = W[L::b13(E) + e];
#pragma unroll
          for (int k = 0; k < 32; ++k) acc = fmaf(W[L::W13 + e * 32 + k], v[k], acc);
          mu_o[e] = fmaxf(acc, 0.f);
        }
      }
    }
    // ---------------- loss and dL/dmu (dune_train.py:300-362) ----------------
    float dmu[kMaxEdges];
    float l_mu = 0.f, l_d = 0.f, l_fa = 0.f, l_fb = 0.f;
    {
      float dd = -prm.dist[pi], fa0 = 0.f, fa1 = 0.f, fb = 0.f;
      float te[kMaxEdges], A0[kMaxEdges], A1[kMaxEdges], ce[kMaxEdges], dl[kMaxEdges];
#pragma unroll
      for (int e = 0; e < kMaxEdges; ++e) {
        te[e] = A0[e] = A1[e] = ce[e] = dl[e] = 0.f;
        if (e < E) {
          const float g0 = prm.G[e][0], g1 = prm.G[e][1];
          te[e] = fmaf(g1, y, g0 * x) - prm.h[e];
          A0[e] = -(cs * g0 - sn * g1);  // fa = (-R G' mu)':  row c of R times G_e
          A1[e] = -(sn * g0 + cs * g1);
          ce[e] = fmaf(A1[e], y, A0[e] * x) + prm.h[e];
          dl[e] = mu_o[e] - prm.mu[(size_t)pi * E + e];
          dd = fmaf(mu_o[e], te[e], dd);  // distance - label_distance
          fa0 = fmaf(dl[e], A0[e], fa0); fa1 = fmaf(dl[e], A1[e], fa1); fb = fmaf(dl[e], ce[e], fb);
          l_mu = fmaf(dl[e], dl[e], l_mu);
        }
      }
      const float inb = 1.0f / (float)nb;
      l_mu *= inb / (float)E; l_d = dd * dd * inb; l_fa = (fa0 * fa0 + fa1 * fa1) * inb * 0.5f; l_fb = fb * fb * inb;
#pragma unroll
      for (int e = 0; e < kMaxEdges; ++e)
        dmu[e] = (e < E && live) ? 2.f * inb * (dl[e] / (float)E + dd * te[e] + 0.5f * (fa0 * A0[e] + fa1 * A1[e]) + fb * ce[e]) : 0.f;
      if (!live) l_mu = l_d = l_fa = l_fb = 0.f;
    }
    {  // batch sums of the four loss terms (warp shuffle, then one atomic per warp into shared doubles)
      float s0 = l_mu, s1 = l_d, s2 = l_fa, s3 = l_fb;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o); s3 += __shfl_xor_sync(0xffffffffu, s3, o);
      }
      if ((tid & 31) == 0) {
        atomicAdd(&loss_acc[0], (double)s0); atomicAdd(&loss_acc[1], (double)s1);
        atomicAdd(&loss_acc[2], (double)s2); atomicAdd(&loss_acc[3], (double)s3);
      }
    }
    if (prm.validate) { __syncthreads(); continue; }

    // ---------------- backward ----------------
    // batch reductions: dW[n][k] = sum_p d[p][n] a[p][k] with d in dbuf and a in the stored layer input; vectors: sum_p d[p][n]
    const int nb4 = (nb + 3) & ~3;  // rows of threads >= nb hold zeros in dbuf: summing up to the next multiple of four is exact
    auto dot4 = [](const float4& u, const float4& w, float c) { return fmaf(u.w, w.w, fmaf(u.z, w.z, fmaf(u.y, w.y, fmaf(u.x, w.x, c)))); };
    auto gemm4 = [&](const float* abuf, float (&g)[4]) {
      float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
      const float* ar = abuf + kcol * kTrainStride;
      const float* dr = dbuf + nrow * kTrainStride;
#pragma unroll 2
      for (int p = 0; p < nb4; p += 4) {
        const float4 a = *reinterpret_cast<const float4*>(ar + p);
        c0 = dot4(*reinterpret_cast<const float4*>(dr + p), a, c0);
        c1 = dot4(*reinterpret_cast<const float4*>(dr + 8 * kTrainStride + p), a, c1);
        c2 = dot4(*reinterpret_cast<const float4*>(dr + 16 * kTrainStride + p), a, c2);
        c3 = dot4(*reinterpret_cast<const float4*>(dr + 24 * kTrainStride + p), a, c3);
      }
      g[0] = c0; g[1] = c1; g[2] = c2; g[3] = c3;
    };
    // sum over the batch of every row of dbuf, returned to the threads tid < 32 (callers use tid < ncols): warp w reduces rows
    // 4 w .. 4 w + 3 (lanes = consecutive points, then a shuffle tree).  Contains two block barriers; called uniformly by all threads.
    auto colsum = [&](int) -> float {
      __syncthreads();  // the previous call's readers are done with `red`
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float* r = dbuf + (4 * nrow + q) * kTrainStride;
        float c = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) c += r[kcol + 32 * i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (kcol == 0) red[4 * nrow + q] = c;
      }
      __syncthreads();
      return tid < 32 ? red[tid] : 0.f;
    };
    float d[32];
    // head: delta6 = dmu * 1[mu > 0]
    {
#pragma unroll
      for (int e = 0; e < kMaxEdges; ++e) dbuf[e * kTrainStride + tid] = (e < E && mu_o[e] > 0.f) ? dmu[e] : 0.f;
      __syncthreads();
      gW13[0] = 0.f;
      if (nrow < E) {  // W13 rows n < E <= 8: one entry per thread (tid < 32 E)
        float c = 0.f;
        const float* abuf = act + 4 * 32 * kTrainStride;
        for (int p = 0; p < nb; ++p) c = fmaf(dbuf[nrow * kTrainStride + p], abuf[kcol * kTrainStride + p], c);
        gW13[0] = c;
      }
      gB13 = colsum(E);
      // d a5 = W13' delta6
#pragma unroll
      for (int k = 0; k < 32; ++k) d[k] = 0.f;
#pragma unroll
      for (int e = 0; e < kMaxEdges; ++e)
        if (e < E) {
          const float de = mu_o[e] > 0.f ? dmu[e] : 0.f;
#pragma unroll
          for (int k = 0; k < 32; ++k) d[k] = fmaf(W[L::W13 + e * 32 + k], de, d[k]);
        }
      __syncthreads();
    }
    // tanh + LayerNorm backward of block (gain off_g, offset off_b, producing linear layer W_l / b_l with stored input `ain`):
    // in: d = dL/da (a = tanh output, stored in `aout`);  out: d = dL/dh (pre-LayerNorm activations);  also the batch sums for gain / offset
    auto ln_tanh_back = [&](const float* aout, const float* ain, int wl, int bl, int off_g, bool first, float& gG, float& gBE) {
      float xh[32];
      if (first) {
#pragma unroll
        for (int j = 0; j < 32; ++j) xh[j] = fmaf(W[wl + 2 * j + 1], y, fmaf(W[wl + 2 * j], x, W[bl + j]));
      } else {
        float in[32];
        train::load_row(ain, tid, in);
        train::linear32(W + wl, W + bl, in, xh);
      }
      const float rstd = train::layer_norm32(xh);
      float s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float a = aout[j * kTrainStride + tid];
        const float dy = live ? d[j] * (1.f - a * a) : 0.f;
        dbuf[j * kTrainStride + tid] = dy * xh[j];  // for the gain
        d[j] = dy;
      }
      __syncthreads();
      gG = colsum(32);
      __syncthreads();
#pragma unroll
      for (int j = 0; j < 32; ++j) dbuf[j * kTrainStride + tid] = d[j];  // for the offset
      __syncthreads();
      gBE = colsum(32);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        d[j] *= W[off_g + j];  // dL/dxhat
        s1 += d[j]; s2 = fmaf(d[j], xh[j], s2);
      }
      s1 *= 1.0f / 32; s2 *= 1.0f / 32;
#pragma unroll
      for (int j = 0; j < 32; ++j) d[j] = rstd * (d[j] - s1 - xh[j] * s2);
      __syncthreads();
    };
    // dense layer backward: d = dL/dh of a 32x32 layer with stored input `ain`; accumulates its weight / bias sums, returns d = W' d
    auto dense_back = [&](const float* ain, int wl, float (&gWl)[4], float& gBl) {
      train::store_row(dbuf, tid, d);
      __syncthreads();
      gemm4(ain, gWl);
      gBl = colsum(32);
      float t[32];
      train::linear32_t(W + wl, d, t);
#pragma unroll
      for (int j = 0; j < 32; ++j) d[j] = t[j];
      __syncthreads();
    };
    float* A1 = act; float* A2 = act + 1 * 32 * kTrainStride; float* A3 = act + 2 * 32 * kTrainStride;
    float* A4 = act + 3 * 32 * kTrainStride; float* A5 = act + 4 * 32 * kTrainStride;
    ln_tanh_back(A5, A4, L::W10, L::B10, L::G11, false, gG11, gBE11);   // d = dL/dh5
    dense_back(A4, L::W10, gW10, gB10);                                 // d = dL/da4
#pragma unroll
    for (int j = 0; j < 32; ++j) d[j] = A4[j * kTrainStride + tid] > 0.f ? d[j] : 0.f;  // ReLU
    dense_back(A3, L::W8, gW8, gB8);                                    // d = dL/da3
    ln_tanh_back(A3, A2, L::W5, L::B5, L::G6, false, gG6, gBE6);        // d = dL/dh3
    dense_back(A2, L::W5, gW5, gB5);                                    // d = dL/da2
#pragma unroll
    for (int j = 0; j < 32; ++j) d[j] = A2[j * kTrainStride + tid] > 0.f ? d[j] : 0.f;
    dense_back(A1, L::W3, gW3, gB3);                                    // d = dL/da1
    ln_tanh_back(A1, nullptr, L::W0, L::B0, L::G1, true, gG1, gBE1);    // d = dL/dh1
    {  // layer 0: dW0[j][c] = sum_p d[p][j] a0[c][p], db0[j] = sum_p d[p][j]
      train::store_row(dbuf, tid, d);
      __syncthreads();
      gW0 = 0.f;
      if (tid < 64) {
        const int j = tid >> 1, c = tid & 1;
        float acc = 0.f;
        for (int p = 0; p < nb; ++p) acc = fmaf(dbuf[j * kTrainStride + p], a0[c * kTrainThreads + p], acc);
        gW0 = acc;
      }
      gB0 = colsum(32);
      __syncthreads();
    }
    // ---------------- Adam (torch.optim.Adam, weight_decay as L2 on the gradient) ----------------
    {
      const long long step = prm.step0 + bi + 1;
      const float bc1 = 1.f - powf(prm.beta1, (float)step), bc2s = sqrtf(1.f - powf(prm.beta2, (float)step));
      const float step_size = prm.lr / bc1;
      auto adam = [&](int idx, float g) {
        const float w = W[idx];
        g = fmaf(prm.weight_decay, w, g);
        const float m = prm.beta1 * prm.adam_m[idx] + (1.f - prm.beta1) * g;
        const float vv = prm.beta2 * prm.adam_v[idx] + (1.f - prm.beta2) * g * g;
        prm.adam_m[idx] = m; prm.adam_v[idx] = vv;
        W[idx] = w - step_size * m / (sqrtf(vv) / bc2s + prm.eps);
      };
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int e = (nrow + 8 * q) * 32 + kcol;
        adam(L::W3 + e, gW3[q]); adam(L::W5 + e, gW5[q]); adam(L::W8 + e, gW8[q]); adam(L::W10 + e, gW10[q]);
      }
      if (nrow < E) adam(L::W13 + nrow * 32 + kcol, gW13[0]);
      if (tid < 64) adam(L::W0 + tid, gW0);
      if (tid < 32) {
        adam(L::B0 + tid, gB0); adam(L::G1 + tid, gG1); adam(L::BE1 + tid, gBE1); adam(L::B3 + tid, gB3); adam(L::B5 + tid, gB5);
        adam(L::G6 + tid, gG6); adam(L::BE6 + tid, gBE6); adam(L::B8 + tid, gB8); adam(L::B10 + tid, gB10);
        adam(L::G11 + tid, gG11); adam(L::BE11 + tid, gBE11);
      }
      if (tid < E) adam(L::b13(E) + tid, gB13);
    }
    __syncthreads();
  }
  if (!prm.validate)
    for (int i = tid; i < nw; i += kTrainThreads) prm.weights[i] = W[i];
  if (tid < 4) prm.losses[tid] = loss_acc[tid];
}

}  // namespace nb
