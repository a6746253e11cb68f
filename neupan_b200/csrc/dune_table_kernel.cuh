// Distance table of the screening pass (NB_OPT_DUNE_SCREEN_TABLE = 1, built by nb_pan when NB_OPT_DUNE_KERNEL = 4 is selected).
//
// The screen's only input per point is p0, the point in the robot frame, and the network and (G, h) are fixed for the lifetime of a
// handle: d(p0) = relu(mu(p0))^T (G p0 - h) is one fixed scalar field of the plane.  It is sampled once on a square grid of cells of
// side h over [-half, half]^2; the screen then costs one 16-byte load (the cell's four corner values), one 4-byte load (its radius)
// and a bilinear interpolation per point instead of the single-pass fp16 network.
//
// Build: (1) dune_table_sample_kernel evaluates the FP32 network (layernorm_tanh / dense32 below) on a grid four times finer
// than the table, (2) dune_table_cell_kernel takes each cell's corners from it and sets the cell's radius to kTableSafety x (the
// largest |bilinear - network| over the 5 x 5 fine samples of the cell + their largest second difference along x or y), plus
// kTableFloor.  The second-difference term covers the ReLU kinks of the network that fall between two fine samples: without it the
// error between the samples reaches twice the radius near the polygon (tests/test_screen_table.py); with it, 0.2 x the radius on the
// shipped checkpoints.  The floor covers the ~1e-6 relative difference between the FP32 network and the exact wgmma network and keeps
// every radius positive.  The radius is checked at run time like the network's: the refine
// kernel compares every candidate's |screened - exact| with half of that candidate's radius.
#pragma once
#include <cuda_fp16.h>

#include "dune_common.cuh"

namespace nb {

constexpr int kTableSub = 4;            // fine samples per cell side used to measure the interpolation error
constexpr float kTableSafety = 4.f;     // radius = kTableSafety x (sample error + second difference) + kTableFloor
constexpr float kTableFloor = 1e-4f;

template <int P>
__device__ __forceinline__ void layernorm_tanh(float (&v)[P][kHidden], const float* __restrict__ g, const float* __restrict__ be) {
#pragma unroll
  for (int p = 0; p < P; ++p) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < kHidden; ++j) s += v[p][j];
    const float mean = s * (1.0f / kHidden);
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < kHidden; ++j) {
      const float d = v[p][j] - mean;
      q = fmaf(d, d, q);
    }
    const float rstd = 1.0f / sqrtf(q * (1.0f / kHidden) + 1e-5f);  // nn.LayerNorm eps, biased variance
#pragma unroll
    for (int j = 0; j < kHidden; ++j) v[p][j] = tanhf(fmaf((v[p][j] - mean) * rstd, g[j], be[j]));
  }
}

// out[p][j] = act(b[j] + sum_k W[j][k] * in[p][k]); W row-major (out, in) in shared memory.
template <int P, bool RELU>
__device__ __forceinline__ void dense32(const float* __restrict__ W, const float* __restrict__ b,
                                        const float (&in)[P][kHidden], float (&out)[P][kHidden]) {
#pragma unroll
  for (int j = 0; j < kHidden; ++j) {
    float acc[P];
#pragma unroll
    for (int p = 0; p < P; ++p) acc[p] = b[j];
#pragma unroll
    for (int k4 = 0; k4 < kHidden / 4; ++k4) {
      const float4 w = reinterpret_cast<const float4*>(W + j * kHidden)[k4];
#pragma unroll
      for (int p = 0; p < P; ++p) {
        acc[p] = fmaf(w.x, in[p][4 * k4 + 0], acc[p]);
        acc[p] = fmaf(w.y, in[p][4 * k4 + 1], acc[p]);
        acc[p] = fmaf(w.z, in[p][4 * k4 + 2], acc[p]);
        acc[p] = fmaf(w.w, in[p][4 * k4 + 3], acc[p]);
      }
    }
#pragma unroll
    for (int p = 0; p < P; ++p) out[p][j] = RELU ? fmaxf(acc[p], 0.f) : acc[p];
  }
}

// out[v * m + u] = d(-half + u hs, -half + v hs), u, v < m, in FP32 (the checkpoint in the packed layout, E <= kMaxEdges)
__global__ void __launch_bounds__(128) dune_table_sample_kernel(const float* __restrict__ weights, const Geometry geo, int m, float half, float hs,
                                                                float* __restrict__ out) {
  using L = WeightLayout;
  __shared__ __align__(16) float sw[L::count(kMaxEdges)];
  const int E = geo.E;
  for (int i = threadIdx.x; i < L::count(E); i += blockDim.x) sw[i] = weights[i];
  __syncthreads();
  const long long total = (long long)m * m;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(q / m), u = (int)(q - (long long)v * m);
    const float x = fmaf((float)u, hs, -half), y = fmaf((float)v, hs, -half);
    float a[1][kHidden], c[1][kHidden];
#pragma unroll
    for (int j = 0; j < kHidden; ++j) a[0][j] = fmaf(sw[L::W0 + 2 * j + 1], y, fmaf(sw[L::W0 + 2 * j], x, sw[L::B0 + j]));
    layernorm_tanh<1>(a, sw + L::G1, sw + L::BE1);
    dense32<1, true>(sw + L::W3, sw + L::B3, a, c);
    dense32<1, false>(sw + L::W5, sw + L::B5, c, a);
    layernorm_tanh<1>(a, sw + L::G6, sw + L::BE6);
    dense32<1, true>(sw + L::W8, sw + L::B8, a, c);
    dense32<1, false>(sw + L::W10, sw + L::B10, c, a);
    layernorm_tanh<1>(a, sw + L::G11, sw + L::BE11);
    float d = 0.f;
#pragma unroll
    for (int e = 0; e < kMaxEdges; ++e) {
      if (e < E) {
        float acc = sw[L::b13(E) + e];
#pragma unroll
        for (int k = 0; k < kHidden; ++k) acc = fmaf(sw[L::W13 + e * kHidden + k], a[0][k], acc);
        const float ge = fmaf(geo.G[e][1], y, geo.G[e][0] * x) - geo.h[e];  // dist = mu^T (G p0 - h)   (dune.py:119-122)
        d = fmaf(fmaxf(acc, 0.f), ge, d);
      }
    }
    out[q] = d;
  }
}

// cell (ix, iy) of n x n from the fine samples f ((kTableSub n + 1)^2): corners, radius; max_ratio (float bits) = the largest
// |bilinear - network| / sum_e |G_e p - h_e| over all fine samples (the quantity nb_pan_read_screen_stats reports for candidates)
__global__ void __launch_bounds__(128) dune_table_cell_kernel(const float* __restrict__ f, int n, float half, float hs, const Geometry geo,
                                                              float4* __restrict__ cell, float* __restrict__ rad, unsigned* max_ratio) {
  const int m = kTableSub * n + 1;
  float worst = 0.f;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n * n; c += gridDim.x * blockDim.x) {
    const int iy = c / n, ix = c - iy * n;
    const float* r0 = f + (size_t)kTableSub * iy * m + (size_t)kTableSub * ix;
    const float4 q = make_float4(r0[0], r0[kTableSub], r0[(size_t)kTableSub * m], r0[(size_t)kTableSub * m + kTableSub]);
    float err = 0.f, d2 = 0.f;
    for (int t = 0; t <= kTableSub; ++t)
      for (int s = 0; s <= kTableSub; ++s) {
        const int u = kTableSub * ix + s, v = kTableSub * iy + t;
        const float* fs = f + (size_t)v * m + u;
        const int ul = u > 0 ? -1 : 0, ur = u < m - 1 ? 1 : 0;                      // grid border: the missing neighbour is the sample itself
        const long long vd = v > 0 ? -(long long)m : 0, vu = v < m - 1 ? (long long)m : 0;
        d2 = fmaxf(d2, fmaxf(fabsf(fs[ul] - 2.f * fs[0] + fs[ur]), fabsf(fs[vd] - 2.f * fs[0] + fs[vu])));
        const float e = fabsf(table_bilerp(q, (float)s / kTableSub, (float)t / kTableSub) - fs[0]);
        const float x = fmaf((float)(kTableSub * ix + s), hs, -half), y = fmaf((float)(kTableSub * iy + t), hs, -half);
        float sa = 0.f;
        for (int k = 0; k < geo.E; ++k) sa += fabsf(fmaf(geo.G[k][1], y, geo.G[k][0] * x) - geo.h[k]);
        err = fmaxf(err, e);
        worst = fmaxf(worst, e / fmaxf(sa, 1e-6f));
      }
    cell[c] = q;
    rad[c] = fmaf(kTableSafety, err + d2, kTableFloor);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) worst = fmaxf(worst, __shfl_xor_sync(0xffffffffu, worst, o));
  if ((threadIdx.x & 31) == 0 && worst > 0.f) atomicMax(max_ratio, __float_as_uint(worst));
}

// Coarse bound table of dune_screen_warp_kernel: coarse cell (u, v) of cn x cn covers the fine cells (ix, iy) with ix >> kCoarseLog = u,
// iy >> kCoarseLog = v (the last row and column cover what is left of the n fine cells) and holds {LB, UB} in fp16 with
//   LB <= fl(table_bilerp(cell, a, b) - rad)  and  UB >= fl(table_bilerp(cell, a, b) + rad)
// for every fine cell it covers and every (a, b) in [0, 1)^2, in the kernel's float arithmetic.
// Margin of table_bilerp: with corners in [lo, hi], X = max |corner| and u = 2^-24, each of d0, d1 = fl(a (c1 - c0) + c0) lies in
// [lo - e, hi + e] with e <= 3.01 u X fused (difference 2 u X, FMA 1.01 u X) or 5.1 u X unfused (+ the product's rounding); the final
// fl(b (d1 - d0) + d0) adds <= 2.01 u X (difference) + 1.01 u X (rounding), + 2.02 u X unfused: at most 10.2 u X in all, so
// m = 16 u X = 2^-20 X, plus FLT_MIN for subnormal results, bounds table_bilerp to [lo - m, hi + m] with or without contraction.
// The bounds then round outward: LB = rd(rd(lo - m) - rad), UB = ru(ru(hi + m) + rad), since fl(d - rad) >= rd(d' - rad) for every d >= d'
// (rounding to nearest is monotone and rd(...) is a float), and the conversion to fp16 rounds down for LB and up for UB.  A zero LB is
// stored as -0 and a zero UB as +0, because orderable() puts -0 below +0.  A fine cell with a non-finite corner or a NaN radius makes
// its coarse cell {-inf, NaN}: every point survives and its key sorts last.
__global__ void __launch_bounds__(128) dune_table_coarse_kernel(const float4* __restrict__ cell, const float* __restrict__ rad, int n, int cn,
                                                                uint32_t* __restrict__ coarse) {
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < cn * cn; q += gridDim.x * blockDim.x) {
    const int v = q / cn, u = q - v * cn;
    const int x0 = u << kCoarseLog, y0 = v << kCoarseLog;
    const int x1 = min(x0 + (1 << kCoarseLog), n), y1 = min(y0 + (1 << kCoarseLog), n);
    float lb = __int_as_float(0x7f800000), ub = -__int_as_float(0x7f800000);
    bool bad = false;
    for (int iy = y0; iy < y1; ++iy)
      for (int ix = x0; ix < x1; ++ix) {
        const float4 c = cell[(size_t)iy * n + ix];
        const float r = rad[(size_t)iy * n + ix];
        const float lo = fminf(fminf(c.x, c.y), fminf(c.z, c.w)), hi = fmaxf(fmaxf(c.x, c.y), fmaxf(c.z, c.w));
        if (!(isfinite(c.x) && isfinite(c.y) && isfinite(c.z) && isfinite(c.w)) || r != r) { bad = true; continue; }
        const float m = fmaf(fmaxf(fabsf(lo), fabsf(hi)), 0x1p-20f, 0x1p-126f);
        lb = fminf(lb, __fsub_rd(__fsub_rd(lo, m), r));
        ub = fmaxf(ub, __fadd_ru(__fadd_ru(hi, m), r));
      }
    __half hl = __float2half_rd(lb), hu = __float2half_ru(ub);
    if (bad) { hl = __float2half_rd(-__int_as_float(0x7f800000)); hu = __float2half(__int_as_float(0x7fc00000)); }
    if (__half2float(hl) == 0.f) hl = __float2half(-0.f);
    if (__half2float(hu) == 0.f) hu = __float2half(0.f);
    coarse[q] = (uint32_t)__half_as_ushort(hl) | ((uint32_t)__half_as_ushort(hu) << 16);
  }
}

}  // namespace nb
