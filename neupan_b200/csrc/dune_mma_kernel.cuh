// DUNE kernel, tensor-core version: same contract as dune_kernel.cuh, ObsPointNet's dense layers on
// the tensor pipe.
//
// Variant 1 of NB_OPT_DUNE_KERNEL (the exact default arithmetic is the wgmma kernel, dune_tc_kernel.cuh).  The network is a
// chain of 32x32 GEMM slices separated by per-row LayerNorm/tanh/ReLU.  With warp-level m16n8k16 the
// accumulator fragment of layer l *is* the A-operand fragment of layer l+1 (same lane <-> (row, column-pair)
// mapping), so 32 points travel through all six layers inside one warp's registers -- no shared-memory
// round trip, no barrier.
//
// Precision: every fp32 operand is split x = hi + lo into two fp16 values (22 significant bits) and
// the product is formed as lo_x*hi_w + hi_x*lo_w + hi_x*hi_w with fp32 accumulation (3 HMMA passes),
// which keeps the layer outputs within ~1e-6 of the fp32 reference; the 2->32 input layer (inputs
// are metres, unbounded) stays on the FP32 FMA pipe.  tanh = 1 - 2/(exp2(2x log2 e) + 1) with
// MUFU.EX2/MUFU.RCP (abs. error ~3e-7).
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "dune_kernel.cuh"  // DuneParams, orderable(), flow()

namespace nb {

// Fragment-ordered weight image built on the host (pan_api.cu: build_mma_image):
//   for each hidden layer L in {3,5,8,10}: uint4 frag[2 ksteps][4 ntiles][32 lanes] = {b0_hi, b1_hi, b0_lo, b1_lo}
//   last layer (13, N padded to 8):        uint4 frag[2 ksteps][1 ntile][32 lanes]
//   then the fp32 vectors: W0 (32x2), b0, g1, be1, b3, b5, g6, be6, b8, b10, g11, be11, b13 (8, zero padded);
//   the LayerNorm gains / offsets g*, be* are stored pre-multiplied by 2*log2(e) (tanh via exp2)
struct MmaImage {
  static constexpr int kHiddenFragU4 = 2 * 4 * 32;  // uint4 per hidden layer
  static constexpr int kLastFragU4 = 2 * 1 * 32;
  static constexpr int kFragU4 = 4 * kHiddenFragU4 + kLastFragU4;  // 1088 uint4 = 17408 B
  // float section offsets (in floats, relative to the float section start)
  static constexpr int W0 = 0, B0 = 64, G1 = 96, BE1 = 128, B3 = 160, B5 = 192, G6 = 224, BE6 = 256, B8 = 288, B10 = 320, G11 = 352,
                       BE11 = 384, B13 = 416, kFloats = 424;
  static constexpr size_t kBytes = (size_t)kFragU4 * 16 + (size_t)kFloats * 4;  // 19104 B
};

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void split_pack(float v0, float v1, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(v0, v1);
  const float2 f = __half22float2(h);
  const __half2 l = __floats2half2_rn(v0 - f.x, v1 - f.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// tanh(x) given a = 2*log2(e)*x (the LayerNorm affine is pre-scaled by that constant in the weight image)
__device__ __forceinline__ float tanh_scaled(float a) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(a));
  const float d = e + 1.0f;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(d));
  return fmaf(-2.0f, r, 1.0f);
}

// A-operand fragments of one 16-row tile for K = 32: [kstep][a0..a3], hi and lo halves
struct AFrag {
  uint32_t hi[2][4];
  uint32_t lo[2][4];
};

// accumulators (n-tile j, c0..c3) -> next layer's A fragments.  c0,c1 = row g, cols 8j+2t,+1; c2,c3 = row g+8.
__device__ __forceinline__ void acc_to_frag(const float (&acc)[4][4], AFrag& f) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int s = j >> 1, o = (j & 1) * 2;
    split_pack(acc[j][0], acc[j][1], f.hi[s][o], f.lo[s][o]);          // a0 / a2 : row g
    split_pack(acc[j][2], acc[j][3], f.hi[s][o + 1], f.lo[s][o + 1]);  // a1 / a3 : row g+8
  }
}

template <int NT, int MT>
__device__ __forceinline__ void dense_mma(const uint4* __restrict__ wfrag, const float* __restrict__ bias, const AFrag (&in)[MT],
                                          float (&acc)[MT][NT][4], int lane) {
  const int t2 = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    const float2 b = *reinterpret_cast<const float2*>(bias + 8 * j + t2);
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      acc[mt][j][0] = b.x; acc[mt][j][1] = b.y; acc[mt][j][2] = b.x; acc[mt][j][3] = b.y;
    }
  }
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      const uint4 w = wfrag[(s * NT + j) * 32 + lane];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        mma16816(acc[mt][j], in[mt].lo[s], w.x, w.y);  // small terms first
        mma16816(acc[mt][j], in[mt].hi[s], w.z, w.w);
        mma16816(acc[mt][j], in[mt].hi[s], w.x, w.y);
      }
    }
}

// LayerNorm (eps 1e-5, biased variance) + tanh on one 16x32 accumulator tile; a row lives in the 4 lanes of a quad
__device__ __forceinline__ void ln_tanh_tile(float (&acc)[4][4], const float* __restrict__ g, const float* __restrict__ be, int lane) {
  const int t2 = (lane & 3) * 2;
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    s0 += acc[j][0] + acc[j][1];
    s1 += acc[j][2] + acc[j][3];
  }
  s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
  s0 += __shfl_xor_sync(0xffffffffu, s0, 2); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
  const float m0 = s0 * (1.0f / 32), m1 = s1 * (1.0f / 32);
  float q0 = 0.f, q1 = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    acc[j][0] -= m0; acc[j][1] -= m0; acc[j][2] -= m1; acc[j][3] -= m1;
    q0 = fmaf(acc[j][0], acc[j][0], q0); q0 = fmaf(acc[j][1], acc[j][1], q0);
    q1 = fmaf(acc[j][2], acc[j][2], q1); q1 = fmaf(acc[j][3], acc[j][3], q1);
  }
  q0 += __shfl_xor_sync(0xffffffffu, q0, 1); q1 += __shfl_xor_sync(0xffffffffu, q1, 1);
  q0 += __shfl_xor_sync(0xffffffffu, q0, 2); q1 += __shfl_xor_sync(0xffffffffu, q1, 2);
  const float r0 = rsqrtf(fmaf(q0, 1.0f / 32, 1e-5f)), r1 = rsqrtf(fmaf(q1, 1.0f / 32, 1e-5f));
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 gg = *reinterpret_cast<const float2*>(g + 8 * j + t2);
    const float2 bb = *reinterpret_cast<const float2*>(be + 8 * j + t2);
    acc[j][0] = tanh_scaled(fmaf(acc[j][0] * r0, gg.x, bb.x));
    acc[j][1] = tanh_scaled(fmaf(acc[j][1] * r0, gg.y, bb.y));
    acc[j][2] = tanh_scaled(fmaf(acc[j][2] * r1, gg.x, bb.x));
    acc[j][3] = tanh_scaled(fmaf(acc[j][3] * r1, gg.y, bb.y));
  }
}

__device__ __forceinline__ void relu_tile(float (&acc)[4][4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[j][c] = fmaxf(acc[j][c], 0.f);
}


// ObsPointNet for MT 16-row tiles held by one warp: robot-frame coordinates in, mu accumulators out
// (pre-ReLU; channels t2, t2+1 of rows g / g+8 in mu[mt][0][0..3]).
template <int MT>
__device__ __forceinline__ void point_net(const uint4* __restrict__ frag, const float* __restrict__ fl, const float (&x0)[MT][2],
                                          const float (&y0)[MT][2], float (&mu)[MT][1][4], int lane) {
  using I = MmaImage;
  const int t2 = (lane & 3) * 2;
  float acc[MT][4][4];
  // layer 0 (2 -> 32) on the FMA pipe, directly in accumulator layout
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 w = *reinterpret_cast<const float4*>(fl + I::W0 + 2 * (8 * j + t2));  // W0[f][0],W0[f][1],W0[f+1][0],W0[f+1][1]
    const float2 bb = *reinterpret_cast<const float2*>(fl + I::B0 + 8 * j + t2);
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      acc[mt][j][0] = fmaf(w.y, y0[mt][0], fmaf(w.x, x0[mt][0], bb.x));
      acc[mt][j][1] = fmaf(w.w, y0[mt][0], fmaf(w.z, x0[mt][0], bb.y));
      acc[mt][j][2] = fmaf(w.y, y0[mt][1], fmaf(w.x, x0[mt][1], bb.x));
      acc[mt][j][3] = fmaf(w.w, y0[mt][1], fmaf(w.z, x0[mt][1], bb.y));
    }
  }
  AFrag a[MT];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) { ln_tanh_tile(acc[mt], fl + I::G1, fl + I::BE1, lane); acc_to_frag(acc[mt], a[mt]); }
  dense_mma<4, MT>(frag + 0 * I::kHiddenFragU4, fl + I::B3, a, acc, lane);
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) { relu_tile(acc[mt]); acc_to_frag(acc[mt], a[mt]); }
  dense_mma<4, MT>(frag + 1 * I::kHiddenFragU4, fl + I::B5, a, acc, lane);
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) { ln_tanh_tile(acc[mt], fl + I::G6, fl + I::BE6, lane); acc_to_frag(acc[mt], a[mt]); }
  dense_mma<4, MT>(frag + 2 * I::kHiddenFragU4, fl + I::B8, a, acc, lane);
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) { relu_tile(acc[mt]); acc_to_frag(acc[mt], a[mt]); }
  dense_mma<4, MT>(frag + 3 * I::kHiddenFragU4, fl + I::B10, a, acc, lane);
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) { ln_tanh_tile(acc[mt], fl + I::G11, fl + I::BE11, lane); acc_to_frag(acc[mt], a[mt]); }
  dense_mma<1, MT>(frag + 4 * I::kHiddenFragU4, fl + I::B13, a, mu, lane);
}

// shared memory: [weight image | per-warp key arrays (N x u64 each)]
__host__ __device__ inline size_t dune_mma_smem_bytes(int N, int warps) {
  return MmaImage::kBytes + (size_t)warps * ((size_t)N * 8) + 16;
}

// One WARP owns one work item (environment b, horizon step t) at a time: it pushes the item's N
// points through the network 32 at a time, keeps only their (distance, index) keys in its private
// slice of shared memory, selects the M smallest with REDUX rounds, then re-evaluates the network
// on those <= 16 points to obtain mu / lambda for the output.  No block-level barrier after the
// weight image is staged: warps drift apart, so the tensor, MUFU, FMA and ALU phases of different
// warps overlap on the SM sub-partitions.
template <int kMT, int kMinBlocks>
__global__ void __launch_bounds__(256, kMinBlocks) dune_mma_kernel(const DuneParams prm, const unsigned char* __restrict__ image) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using I = MmaImage;
  const uint4* frag = reinterpret_cast<const uint4*>(smem_raw);
  const float* fl = reinterpret_cast<const float*>(smem_raw + (size_t)I::kFragU4 * 16);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nthreads = blockDim.x, nwarps = nthreads >> 5;
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw + I::kBytes) + (size_t)warp * prm.N;
  const int g = lane >> 2, tq = lane & 3, t2 = tq * 2;
  for (int i = tid; i < (int)(I::kBytes / 16); i += nthreads) reinterpret_cast<uint4*>(smem_raw)[i] = reinterpret_cast<const uint4*>(image)[i];
  __syncthreads();

  const int T1 = prm.T + 1, N = prm.N, M = prm.M, E = prm.geo.E;
  const int items = prm.B * T1;
  float Gx[2], Gy[2], hh[2];  // geometry rows of this lane's two output channels
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const int e = t2 + c;
    Gx[c] = e < E ? prm.geo.G[e][0] : 0.f;
    Gy[c] = e < E ? prm.geo.G[e][1] : 0.f;
    hh[c] = e < E ? prm.geo.h[e] : 0.f;
  }

  for (int item = blockIdx.x * nwarps + warp; item < items; item += gridDim.x * nwarps) {
    const int b = item / T1, t = item - b * T1;
    if (prm.active && prm.active[b] == 0) continue;
    int n = prm.num_points ? prm.num_points[b] : N;
    n = n < 0 ? 0 : (n > N ? N : n);
    const int cnt = n < M ? n : M;
    if (t == 0 && lane == 0) {
      prm.sel_count[b] = cnt;
      if (n == 0 && prm.min_dist) prm.min_dist[b] = __int_as_float(0x7f800000);
    }
    if (n == 0) continue;

    const float* ns = prm.nom_s + (size_t)b * 3 * T1;
    const float sx = ns[t], sy = ns[T1 + t], th = ns[2 * T1 + t];
    const float cs = cosf(th), sn = sinf(th);
    const float* px = prm.points + (size_t)b * 2 * N;
    const float* py = px + N;
    const float* vx = prm.velocities ? prm.velocities + (size_t)b * 2 * N : nullptr;
    const float* vy = vx ? vx + N : nullptr;
    auto robot_frame = [&](int i, float& gx, float& gy, float& x0, float& y0) {
      gx = px[i]; gy = py[i];
      if (vx) {
        gx = flow(gx, vx[i], prm.dt, t);
        gy = flow(gy, vy[i], prm.dt, t);
      }
      const float dx = gx - sx, dy = gy - sy;  // p0 = R^T (p_t - trans)   (pan.py:210)
      x0 = fmaf(cs, dx, sn * dy);
      y0 = fmaf(cs, dy, -(sn * dx));
    };

    // ---- phase 1: distances of all points, 32 per pass, everything in registers ------------------
    constexpr int kPts = 16 * kMT;  // points per pass
    const int chunks = (n + kPts - 1) / kPts;
#pragma unroll 1
    for (int ch = 0; ch < chunks; ++ch) {
      const int base = ch * kPts;
      float x0[kMT][2], y0[kMT][2];
#pragma unroll
      for (int mt = 0; mt < kMT; ++mt)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          int i = base + mt * 16 + r * 8 + g;
          i = i < n ? i : n - 1;
          float gx, gy;
          robot_frame(i, gx, gy, x0[mt][r], y0[mt][r]);
        }
      float mu[kMT][1][4];
      point_net<kMT>(frag, fl, x0, y0, mu, lane);
      // distance = mu^T (G p0 - h): quad-reduce; lane (g, tq) keeps the key of point (mt, r) = (tq>>1, tq&1)
      float myd = 0.f;
#pragma unroll
      for (int mt = 0; mt < kMT; ++mt)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float m0 = fmaxf(mu[mt][0][2 * r], 0.f), m1 = fmaxf(mu[mt][0][2 * r + 1], 0.f);
          float d = m0 * (fmaf(Gy[0], y0[mt][r], Gx[0] * x0[mt][r]) - hh[0]);
          d = fmaf(m1, fmaf(Gy[1], y0[mt][r], Gx[1] * x0[mt][r]) - hh[1], d);
          d += __shfl_xor_sync(0xffffffffu, d, 1);
          d += __shfl_xor_sync(0xffffffffu, d, 2);
          if (mt * 2 + r == tq) myd = d;
        }
      // lane (g, tq) stores the key of point (mt, r) = (tq>>1, tq&1); with one tile only tq < 2 own a point
      const int i = base + (tq >> 1) * 16 + (tq & 1) * 8 + g;
      if (i < n && (tq >> 1) < kMT) keys[i] = ((unsigned long long)orderable(myd) << 32) | (unsigned)i;
    }
    __syncwarp();

    // ---- phase 2: the M smallest keys, ascending (ties -> lower index) ------------------------------
    unsigned sel_idx = 0, sel_ord = 0xFFFFFFFFu;  // lane m holds the m-th closest point
#pragma unroll 1
    for (int m = 0; m < cnt; ++m) {
      unsigned bd = 0xFFFFFFFFu, bi = 0xFFFFFFFFu;
      for (int i = lane; i < n; i += 32) {
        const uint2 k = *reinterpret_cast<const uint2*>(keys + i);  // .x = index, .y = orderable distance
        if (k.y < bd) { bd = k.y; bi = k.x; }
      }
      const unsigned md = __reduce_min_sync(0xffffffffu, bd);
      const unsigned mi = __reduce_min_sync(0xffffffffu, bd == md ? bi : 0xFFFFFFFFu);
      if (md != 0xFFFFFFFFu && bd == md && bi == mi) keys[mi] = ~0ull;  // the owner lane retires it
      if (lane == m) { sel_idx = mi; sel_ord = md; }
      __syncwarp();
    }

    // ---- phase 3: mu / lambda of the selected points: one more 16-row tile (row m = m-th closest) ----
    {
      float x0[1][2], y0[1][2], gxs[2], gys[2];
      int rows[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int row = r * 8 + g;
        unsigned idx = __shfl_sync(0xffffffffu, sel_idx, row < cnt ? row : 0);
        if (idx >= (unsigned)n) idx = 0;  // all-NaN distances: keep the access in range
        rows[r] = row;
        robot_frame((int)idx, gxs[r], gys[r], x0[0][r], y0[0][r]);
      }
      float mu[1][1][4];
      point_net<1>(frag, fl, x0, y0, mu, lane);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float m0 = fmaxf(mu[0][0][2 * r], 0.f), m1 = fmaxf(mu[0][0][2 * r + 1], 0.f);
        // lam = ((-R) G^T) mu   (dune.py:89), partial sums over this lane's two channels, then the quad
        float lx = fmaf(fmaf(sn, Gy[1], -cs * Gx[1]), m1, fmaf(sn, Gy[0], -cs * Gx[0]) * m0);
        float ly = fmaf(fmaf(-cs, Gy[1], -sn * Gx[1]), m1, fmaf(-cs, Gy[0], -sn * Gx[0]) * m0);
        lx += __shfl_xor_sync(0xffffffffu, lx, 1); ly += __shfl_xor_sync(0xffffffffu, ly, 1);
        lx += __shfl_xor_sync(0xffffffffu, lx, 2); ly += __shfl_xor_sync(0xffffffffu, ly, 2);
        const unsigned ord = __shfl_sync(0xffffffffu, sel_ord, rows[r] < cnt ? rows[r] : 0);
        if (rows[r] < cnt) {
          const size_t o = ((size_t)b * T1 + t) * M + rows[r];
          if (t2 < E) prm.sel_mu[o * E + t2] = m0;
          if (t2 + 1 < E) prm.sel_mu[o * E + t2 + 1] = m1;
          if (tq == 0) {
            const uint32_t u = (ord & 0x80000000u) ? (ord & 0x7fffffffu) : ~ord;
            const float d = __uint_as_float(u);
            prm.sel_lam[o * 2 + 0] = lx; prm.sel_lam[o * 2 + 1] = ly;
            prm.sel_pts[o * 2 + 0] = gxs[r]; prm.sel_pts[o * 2 + 1] = gys[r];
            prm.sel_dist[o] = d;
            if (t == 0 && rows[r] == 0 && prm.min_dist) prm.min_dist[b] = d;  // dune.py:97-98
          }
        }
      }
    }
    __syncwarp();
  }
}

}  // namespace nb
