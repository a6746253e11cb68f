// Screening pass of DUNE on the warp-level tensor pipe (mma.sync m16n8k16, fp16 in / fp32 accumulate): same contract, same
// candidate lists and the same operand image as dune_screen_kernel (dune_screen_kernel.cuh), different execution shape.
//
// Why a second shape for this one pass.  The screening network is SINGLE-pass fp16 (no hi/lo split): per 32-wide layer and 128
// points it needs 3 wgmma of 64x32x16 per half tile -- a tiny amount of tensor work -- but dune_screen_kernel pays a round trip
// through shared memory five times per tile: operand store, block barrier, MMA wait, fp32 row load.  With mma.sync m16n8k16 the
// accumulator fragment of layer l IS the A fragment of layer l+1 (same lane <-> (row, column pair) map), so 32 points travel
// through all six layers inside one warp's registers: no shared-memory tile, no block barrier inside the network, warps drift
// freely and the MUFU (tanh), FMA, ALU and tensor phases of the four warps of a scheduler overlap.  The exact path (3 passes)
// keeps the warpgroup kernels (dune_refine_kernel / dune_tcp_kernel).
//
// Two kernels: dune_screen_warp_kernel (clouds of <= 512 points: one warp per (environment, step) item, see its comment) and
// dune_screen_mma_kernel (513..1024 points: CTA = 4 warps = one item at a time; pass p, warp w: points [128 p + 32 w, +32)).
// The network tile is the same in both: 32 points as two m16 tiles.
// Lane (g = lane >> 2, tq = lane & 3) holds rows g, g+8 (tile 0), g, g+8 (tile 1) -- "row slots" 0..3 = local points g + 8 r --
// and columns 8 j + 2 tq, +1 (j = 0..3) of every 32-wide activation; it OWNS local point 8 tq + g (coordinates in, key out), so
// the four row slots of a quad are exactly the points its four lanes own (one shuffle each way, no shared memory).
// LayerNorm: per-row sum of squares by a transposing quad reduction (3 shuffles: lane tq ends with the total of row slot tq),
// one MUFU.RSQ per lane, 4 shuffles to hand the four factors round.  The inputs arrive centred (host image), see ln_tanh_screen.
#pragma once
#include "dune_screen_kernel.cuh"

namespace nb {

namespace sm {

using tc::f2;

#ifndef NB_WHATIF
#define NB_WHATIF 0  // timing experiments only (wrong results): 1 = no MUFU.TANH, 2 = no HMMA, 4 = no selection, 8 = no LayerNorm scale math,
                     // 16 = every point of dune_screen_warp_kernel's table branch gathers cell 0 (a broadcast: no L2 traffic) and takes
                     // |x| + |y| in the robot frame as its distance, so that the candidate lists keep a realistic length
#endif

constexpr int kFragBytes = 5 * 2 * 2 * 32 * 16;  // B fragments, [layer][k-step][n-tile pair][lane] uint4 = {b0,b1 (tile 2jp), b0,b1 (2jp+1)}
enum { V_W0X, V_W0Y, V_B0, V_G1, V_BE1, V_G6, V_BE6, V_G11, V_BE11, kVecs };
constexpr int kVecBytes = kVecs * 32 * 4;  // the fp32 vectors, permuted so that a lane's 8 columns are contiguous: [tq][j][h]
// the dense layers' biases as ready-made C fragments: [layer][tq][j] = {b[8j+2tq], b[8j+2tq+1], same, same} (rows g and g+8 share them),
// so that one LDS.128 delivers the aligned register quad HMMA wants (building it from a pair costs 4 moves per HMMA)
constexpr int kBiasQBytes = 5 * 4 * 4 * 16;

// D = A.B + C: the first k-step of a layer (C = the bias fragment of the lane's column pair, the same for both rows)
__device__ __forceinline__ void mma_init(f2& d01, f2& d23, const uint32_t (&a)[4], uint32_t b0, uint32_t b1, const float4& c) {
  if (NB_WHATIF & 2) {
    d01 = tc::pku(a[0] ^ b0, a[1] ^ __float_as_uint(c.x));
    d23 = tc::pku(a[2] ^ b1, a[3] ^ __float_as_uint(c.y));
    return;
  }
  asm("{\n\t.reg .f32 e0, e1, e2, e3;\n\t"
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {e0, e1, e2, e3}, {%2, %3, %4, %5}, {%6, %7}, {%8, %9, %10, %11};\n\t"
      "mov.b64 %0, {e0, e1};\n\tmov.b64 %1, {e2, e3};\n\t}"
      : "=l"(d01), "=l"(d23)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "f"(c.x), "f"(c.y), "f"(c.z), "f"(c.w));
}
__device__ __forceinline__ void mma_acc(f2& d01, f2& d23, const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if (NB_WHATIF & 2) {
    d01 ^= tc::pku(a[0] ^ b0, a[1]);
    d23 ^= tc::pku(a[2] ^ b1, a[3]);
    return;
  }
  asm("{\n\t.reg .f32 e0, e1, e2, e3;\n\t"
      "mov.b64 {e0, e1}, %0;\n\tmov.b64 {e2, e3}, %1;\n\t"
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {e0, e1, e2, e3}, {%2, %3, %4, %5}, {%6, %7}, {e0, e1, e2, e3};\n\t"
      "mov.b64 %0, {e0, e1};\n\tmov.b64 %1, {e2, e3};\n\t}"
      : "+l"(d01), "+l"(d23)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// v[r] = this lane's partial of row slot r; returns the quad total of row slot tq (lane tq of the quad)
__device__ __forceinline__ float quad_transpose_sum(const float (&v)[4], int tq) {
  const bool b0 = tq & 1, b1 = tq & 2;
  float k0 = b0 ? v[1] : v[0], s0 = b0 ? v[0] : v[1];
  float k1 = b0 ? v[3] : v[2], s1 = b0 ? v[2] : v[3];
  k0 += __shfl_xor_sync(0xffffffffu, s0, 1);
  k1 += __shfl_xor_sync(0xffffffffu, s1, 1);
  const float k = b1 ? k1 : k0, s = b1 ? k0 : k1;
  return k + __shfl_xor_sync(0xffffffffu, s, 2);
}

// LayerNorm (centred inputs, eps 1e-5, biased variance) + tanh (MUFU.TANH) on the lane's 4 row slots x 8 columns; the result is
// written as the A fragments of the next layer: a[m-tile][k-step][a0..a3]
__device__ __forceinline__ void ln_tanh_frag(const f2 (&acc)[4][4], const float* __restrict__ vg, const float* __restrict__ vb, int lane,
                                             uint32_t (&a)[2][2][4]) {
  float q[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    f2 s = tc::mul2(acc[r][0], acc[r][0]);
    s = tc::fma2(acc[r][1], acc[r][1], s);
    s = tc::fma2(acc[r][2], acc[r][2], s);
    s = tc::fma2(acc[r][3], acc[r][3], s);
    float lo, hi;
    tc::upk(s, lo, hi);
    q[r] = lo + hi;
  }
  const float qq = quad_transpose_sum(q, lane & 3);
  float rs;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(rs) : "f"(fmaf(qq, 1.0f / 32, 1e-5f)));
  const ulonglong2 g01 = *reinterpret_cast<const ulonglong2*>(vg), g23 = *reinterpret_cast<const ulonglong2*>(vg + 4);
  const ulonglong2 b01 = *reinterpret_cast<const ulonglong2*>(vb), b23 = *reinterpret_cast<const ulonglong2*>(vb + 4);
  const f2 gg[4] = {g01.x, g01.y, g23.x, g23.y}, bb[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const float rr = __shfl_sync(0xffffffffu, rs, (lane & ~3) | r);
    const f2 r2 = tc::pk(rr, rr);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float a0, a1, t0, t1;
      if (NB_WHATIF & 8) tc::upk(tc::add2(acc[r][j], r2), a0, a1);
      else tc::upk(tc::fma2(tc::mul2(acc[r][j], r2), gg[j], bb[j]), a0, a1);
      if (NB_WHATIF & 1) { t0 = a0; t1 = a1; }
      else {
        asm("tanh.approx.f32 %0, %1;" : "=f"(t0) : "f"(a0));
        asm("tanh.approx.f32 %0, %1;" : "=f"(t1) : "f"(a1));
      }
      asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(a[r >> 1][j >> 1][(j & 1) * 2 + (r & 1)]) : "f"(t1), "f"(t0));
    }
  }
}

__device__ __forceinline__ void relu_frag(const f2 (&acc)[4][4], uint32_t (&a)[2][2][4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float a0, a1;
      tc::upk(acc[r][j], a0, a1);
      asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(a[r >> 1][j >> 1][(j & 1) * 2 + (r & 1)]) : "f"(a1), "f"(a0));
    }
}

// one dense layer (K = 32) for both m-tiles: NT n-tiles of 8 columns; wl = the layer's fragments + lane, bq = its bias fragments + 4 tq
template <int NT>
__device__ __forceinline__ void dense_frag(const uint4* __restrict__ wl, const float4* __restrict__ bq, const uint32_t (&a)[2][2][4],
                                           f2 (&acc)[4][NT]) {
  float4 bj[NT];
#pragma unroll
  for (int j = 0; j < NT; ++j) bj[j] = bq[j];
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int jp = 0; jp < (NT + 1) / 2; ++jp) {
      const uint4 w = wl[(s * 2 + jp) * 32];
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int j = 2 * jp + jj;
        if (j < NT) {
          const uint32_t b0 = jj ? w.z : w.x, b1 = jj ? w.w : w.y;
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            if (s == 0) mma_init(acc[2 * mt][j], acc[2 * mt + 1][j], a[mt][0], b0, b1, bj[j]);
            else mma_acc(acc[2 * mt][j], acc[2 * mt + 1][j], a[mt][1], b0, b1);
          }
        }
      }
    }
}

// operand staging by `nthreads` threads: the screen image of dune_screen_kernel (K-major wgmma layout, hi halves) re-ordered into
// mma.sync B fragments, the permuted vectors and the bias fragments
__device__ __forceinline__ void stage_operands(const unsigned char* __restrict__ image, uint4* wfrag, float* vec, float4* biasq, int tid, int nthreads) {
  using I = TcImage;
  uint32_t* wf = reinterpret_cast<uint32_t*>(wfrag);
  for (int x = tid; x < kFragBytes / 4; x += nthreads) {
    const int c = x & 3, ln = (x >> 2) & 31, jp = (x >> 7) & 1, s = (x >> 8) & 1, l = x >> 9;
    const int n = 8 * (2 * jp + (c >> 1)) + (ln >> 2), k = 16 * s + 2 * (ln & 3) + 8 * (c & 1);
    const size_t off = (size_t)l * I::kLayerStride + (size_t)(k / 16) * 1024 + ((k % 16) / 8) * 512 + (n / 8) * 128 + (n % 8) * 16 + (k % 8) * 2;
    wf[x] = *reinterpret_cast<const uint32_t*>(image + off);
  }
  const float* fl = reinterpret_cast<const float*>(image + I::kFloatOff);
  for (int x = tid; x < kVecs * 32; x += nthreads) {
    const int v = x >> 5, e = x & 31, q = e >> 3, j = (e >> 1) & 3, h = e & 1;
    const int src = v == V_W0X ? I::W0X : v == V_W0Y ? I::W0Y : v == V_B0 ? I::B0 : I::G1 + 32 * (v - V_G1);
    vec[x] = fl[src + 8 * j + 2 * q + h];
  }
  for (int x = tid; x < 5 * 4 * 4; x += nthreads) {  // [layer][tq][j]
    const int l = x >> 4, q = (x >> 2) & 3, j = x & 3;
    const float bx = fl[I::BH + 32 * l + 8 * j + 2 * q], by = fl[I::BH + 32 * l + 8 * j + 2 * q + 1];
    biasq[x] = make_float4(bx, by, bx, by);
  }
}

// The screening network on one 32-point tile, all six layers in the warp's registers.  (x0, y0) = the robot-frame coordinates of the
// lane's own point (local point 8 tq + g of the tile; zeros for rows beyond the cloud); returns that point's d~.  wl, vq, bqq: the
// lane's views of the staged operands.
__device__ __forceinline__ float tile_network(const Geometry& geo, float x0, float y0, int lane, const uint4* __restrict__ wl,
                                              const float* __restrict__ vq, const float4* __restrict__ bqq) {
  float xr[4], yr[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    xr[r] = __shfl_sync(0xffffffffu, x0, (lane & ~3) | r);
    yr[r] = __shfl_sync(0xffffffffu, y0, (lane & ~3) | r);
  }
  f2 acc[4][4];
  uint32_t a[2][2][4];
  {  // layer 0 (2 -> 32) on the FMA pipe, directly in accumulator layout
    const ulonglong2 wx01 = *reinterpret_cast<const ulonglong2*>(vq + 32 * V_W0X), wx23 = *reinterpret_cast<const ulonglong2*>(vq + 32 * V_W0X + 4);
    const ulonglong2 wy01 = *reinterpret_cast<const ulonglong2*>(vq + 32 * V_W0Y), wy23 = *reinterpret_cast<const ulonglong2*>(vq + 32 * V_W0Y + 4);
    const ulonglong2 b01 = *reinterpret_cast<const ulonglong2*>(vq + 32 * V_B0), b23 = *reinterpret_cast<const ulonglong2*>(vq + 32 * V_B0 + 4);
    const f2 wx[4] = {wx01.x, wx01.y, wx23.x, wx23.y}, wy[4] = {wy01.x, wy01.y, wy23.x, wy23.y}, bb[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const f2 x2 = tc::pk(xr[r], xr[r]), y2 = tc::pk(yr[r], yr[r]);
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[r][j] = tc::fma2(wy[j], y2, tc::fma2(wx[j], x2, bb[j]));
    }
  }
  ln_tanh_frag(acc, vq + 32 * V_G1, vq + 32 * V_BE1, lane, a);
  dense_frag<4>(wl + 0 * 128, bqq + 16 * 0, a, acc);
  relu_frag(acc, a);
  dense_frag<4>(wl + 1 * 128, bqq + 16 * 1, a, acc);
  ln_tanh_frag(acc, vq + 32 * V_G6, vq + 32 * V_BE6, lane, a);
  dense_frag<4>(wl + 2 * 128, bqq + 16 * 2, a, acc);
  relu_frag(acc, a);
  dense_frag<4>(wl + 3 * 128, bqq + 16 * 3, a, acc);
  ln_tanh_frag(acc, vq + 32 * V_G11, vq + 32 * V_BE11, lane, a);
  f2 mu[4][1];
  dense_frag<1>(wl + 4 * 128, bqq + 16 * 4, a, mu);

  // head: d~ = relu(mu)^T (G p0 - h): partial over the lane's two channels for each row slot, transposing quad reduction
  // geometry rows of the lane's two head channels (zero beyond E: their partial distance is 0)
  const int e0 = 2 * (lane & 3), e1 = e0 + 1;
  const float gx0 = e0 < geo.E ? geo.G[e0][0] : 0.f, gy0 = e0 < geo.E ? geo.G[e0][1] : 0.f, h0 = e0 < geo.E ? geo.h[e0] : 0.f;
  const float gx1 = e1 < geo.E ? geo.G[e1][0] : 0.f, gy1 = e1 < geo.E ? geo.G[e1][1] : 0.f, h1 = e1 < geo.E ? geo.h[e1] : 0.f;
  float dp[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    float m0, m1;
    tc::upk(mu[r][0], m0, m1);
    const float ge0 = fmaf(gy0, yr[r], gx0 * xr[r]) - h0, ge1 = fmaf(gy1, yr[r], gx1 * xr[r]) - h1;
    dp[r] = fmaf(fmaxf(m1, 0.f), ge1, fmaxf(m0, 0.f) * ge0);
  }
  return quad_transpose_sum(dp, lane & 3);  // the lane's own point
}

// the error radius the network screen assumes for the point (x0, y0): c_mu sum_e |G_e p0 - h_e| + 1e-4
__device__ __forceinline__ float network_radius(const DuneParams& prm, float x0, float y0) {
  float sa = 0.f;
#pragma unroll
  for (int e = 0; e < kMaxEdges; ++e)
    if (e < prm.geo.E) sa += fabsf(fmaf(prm.geo.G[e][1], y0, prm.geo.G[e][0] * x0) - prm.geo.h[e]);
  return fmaf(prm.c_mu, sa, 1e-4f);
}

}  // namespace sm

// shared memory: B fragments | permuted vectors | bias fragments | raw points of the item in flight (x | y | vx | vy, N floats each) |
// per-warp upper-bound candidates (4 M x 4)
__host__ __device__ inline size_t dune_screen_mma_smem_bytes(int N, int M) {
  return (size_t)sm::kFragBytes + sm::kVecBytes + sm::kBiasQBytes + (size_t)N * 16 + (size_t)4 * M * 4 + 64;
}

// Clouds of 513..1024 points (smaller ones take dune_screen_warp_kernel below, larger ones dune_screen_kernel, whose shared-memory key
// arrays have no size limit).  kP = the most 128-point passes an item can need: every thread keeps the bounds of its <= kP points in
// registers, with the point's index in the low kIdxBits bits of the key.
__global__ void __launch_bounds__(128, 4) dune_screen_mma_kernel(const DuneParams prm, const unsigned char* __restrict__ image) {
  constexpr int kP = 8;
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  using I = TcImage;
  uint4* wfrag = reinterpret_cast<uint4*>(smem_dyn);
  float* vec = reinterpret_cast<float*>(smem_dyn + sm::kFragBytes);
  float4* biasq = reinterpret_cast<float4*>(smem_dyn + sm::kFragBytes + sm::kVecBytes);
  float* raw = reinterpret_cast<float*>(smem_dyn + sm::kFragBytes + sm::kVecBytes + sm::kBiasQBytes);
  uint32_t* c32 = reinterpret_cast<uint32_t*>(raw + (size_t)4 * prm.N);
  __shared__ int cnt_s[2];
  __shared__ int list_s[kCandMax];
  __shared__ float ldt_s[kCandMax], lrad_s[kCandMax];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, tq = lane & 3;
  // ---- operand staging: the screen image of dune_screen_kernel (K-major wgmma layout, hi halves) re-ordered into mma.sync B fragments
  {
    uint32_t* wf = reinterpret_cast<uint32_t*>(wfrag);
    for (int x = tid; x < sm::kFragBytes / 4; x += 128) {
      const int c = x & 3, ln = (x >> 2) & 31, jp = (x >> 7) & 1, s = (x >> 8) & 1, l = x >> 9;
      const int n = 8 * (2 * jp + (c >> 1)) + (ln >> 2), k = 16 * s + 2 * (ln & 3) + 8 * (c & 1);
      const size_t off = (size_t)l * I::kLayerStride + (size_t)(k / 16) * 1024 + ((k % 16) / 8) * 512 + (n / 8) * 128 + (n % 8) * 16 + (k % 8) * 2;
      wf[x] = *reinterpret_cast<const uint32_t*>(image + off);
    }
    const float* fl = reinterpret_cast<const float*>(image + I::kFloatOff);
    for (int x = tid; x < sm::kVecs * 32; x += 128) {
      const int v = x >> 5, e = x & 31, q = e >> 3, j = (e >> 1) & 3, h = e & 1;
      const int src = v == sm::V_W0X ? I::W0X : v == sm::V_W0Y ? I::W0Y : v == sm::V_B0 ? I::B0 : I::G1 + 32 * (v - sm::V_G1);
      vec[x] = fl[src + 8 * j + 2 * q + h];
    }
    for (int x = tid; x < 5 * 4 * 4; x += 128) {  // [layer][tq][j]
      const int l = x >> 4, q = (x >> 2) & 3, j = x & 3;
      const float bx = fl[I::BH + 32 * l + 8 * j + 2 * q], by = fl[I::BH + 32 * l + 8 * j + 2 * q + 1];
      biasq[x] = make_float4(bx, by, bx, by);
    }
    if (tid < 2) cnt_s[tid] = 0;
  }
  __syncthreads();
  const uint4* wl = wfrag + lane;
  const float* vq = vec + 8 * tq;
  const float4* bqq = biasq + 4 * tq;

  const int T1 = prm.T + 1, N = prm.N, M = prm.M, E = prm.geo.E;
  const int items = prm.B * T1;
  // geometry rows of this lane's two head channels (zero beyond E: their partial distance is 0)
  const int e0 = 2 * tq, e1 = 2 * tq + 1;
  const float gx0 = e0 < E ? prm.geo.G[e0][0] : 0.f, gy0 = e0 < E ? prm.geo.G[e0][1] : 0.f, h0 = e0 < E ? prm.geo.h[e0] : 0.f;
  const float gx1 = e1 < E ? prm.geo.G[e1][0] : 0.f, gy1 = e1 < E ? prm.geo.G[e1][1] : 0.f, h1 = e1 < E ? prm.geo.h[e1] : 0.f;
  const int own0 = 32 * warp + 8 * tq + g;  // the lane's point in pass 0 (pass p: + 128 p)
  constexpr int kIdxBits = 10;
  constexpr uint32_t kIdxMask = (1u << kIdxBits) - 1u;
  // smallest value above k whose low kIdxBits bits carry the point's index: keys become unique (a REDUX round removes exactly one entry);
  // rounding an upper bound UP only widens the candidate set
  auto unique_key = [&](uint32_t k, int idx) -> uint32_t { return ((min(k, 0xFFFFF000u) + (kIdxMask + 1u)) & ~kIdxMask) | (uint32_t)idx; };

  // The raw point data of an item are copied asynchronously (cp.async, each thread exactly the <= 4 entries it reads itself: no
  // barrier) -- for the NEXT item as soon as this thread has read its last point of the current one.
  int staged = -1;
  auto stage_points = [&](int it) -> bool {
    const int bb = it / T1;
    if (prm.skip_t0 && it == bb * T1) return false;
    int nn = prm.num_points ? prm.num_points[bb] : N;
    nn = nn > N ? N : nn;
    if ((nn <= kCandMax && !prm.calibrate) || nn <= 0) return false;
    const float* px = prm.points + (size_t)bb * 2 * N;
    const float* vx = prm.velocities ? prm.velocities + (size_t)bb * 2 * N : nullptr;
#pragma unroll
    for (int j = 0; j < kP; ++j) {
      const int i = own0 + 128 * j;
      if (i < nn) {
        tc::cp_async4(raw + i, px + i);
        tc::cp_async4(raw + N + i, px + N + i);
        if (vx) {
          tc::cp_async4(raw + 2 * N + i, vx + i);
          tc::cp_async4(raw + 3 * N + i, vx + N + i);
        }
      }
    }
    return true;
  };

  int par = 0;  // which of the two candidate counters this item uses (the other one is reset meanwhile)
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int b = item / T1, t = item - b * T1;
    if (prm.skip_t0 && t == 0) {  // same inputs as in the previous PAN iteration: its outputs stand
      if (tid == 0) prm.cand_cnt[item] = 0;
      continue;
    }
    int32_t* out_idx = prm.cand_idx + (size_t)item * kCandMax;
    float* out_dt = prm.cand_dt + (size_t)item * kCandMax;
    const int act = prm.active ? prm.active[b] : 1;
    int n = prm.num_points ? prm.num_points[b] : N;
    const tc::ItemFrame fr = tc::item_frame(prm, b, t);
    if (act == 0) {
      if (tid == 0) prm.cand_cnt[item] = 0;
      continue;
    }
    n = n < 0 ? 0 : (n > N ? N : n);
    const int cnt = n < M ? n : M;
    if (t == 0 && tid == 0) {
      prm.sel_count[b] = cnt;
      if (n == 0 && prm.min_dist) prm.min_dist[b] = __int_as_float(0x7f800000);
    }
    if (n <= kCandMax && !prm.calibrate) {  // nothing to screen: every point is a candidate
      if (tid < n) { out_idx[tid] = tid; out_dt[tid] = __int_as_float(0x7fc00000); }
      if (tid == 0) { prm.cand_cnt[item] = n; tc::refine_append(prm, item, n); }
      continue;
    }
    if (staged != item) {
      tc::cp_async_wait_all();  // an abandoned copy (its item was skipped) must not land after this one
      stage_points(item);
      staged = item;
    }
    tc::cp_async_wait_all();
    // the bounds of the thread's points: a shift register (newest first); the point's index rides in the low 9 bits of the key
    uint32_t kk[kP];
    float ll[kP], dd[kP];
#pragma unroll
    for (int j = 0; j < kP; ++j) { kk[j] = 0xFFFFFFFFu; ll[j] = 0.f; dd[j] = 0.f; }

#pragma unroll 1
    for (int base = 32 * warp; base < n; base += 128) {  // this warp's 32-point tiles
      const int i = base + 8 * tq + g;
      float x0 = 0.f, y0 = 0.f;
      if (i < n) {  // rows beyond n run on zeros (their results are never looked at)
        float gx = raw[i], gy = raw[N + i];
        if (fr.vx) {
          gx = flow(gx, raw[2 * N + i], fr.dt, fr.t);
          gy = flow(gy, raw[3 * N + i], fr.dt, fr.t);
        }
        const float dx = gx - fr.sx, dy = gy - fr.sy;
        x0 = fmaf(fr.cs, dx, fr.sn * dy);
        y0 = fmaf(fr.cs, dy, -(fr.sn * dx));
      }
      // the distance table where it covers the point (rows beyond n need nothing); the warp runs the network on its tile when any
      // of its points lies outside the table, or when there is no table
      float d = 0.f, eps = 0.f;
      const bool hit = prm.tab_cell != nullptr && (i >= n || table_lookup(prm, x0, y0, d, eps));
      if (!__all_sync(0xffffffffu, hit)) {
        float xr[4], yr[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          xr[r] = __shfl_sync(0xffffffffu, x0, (lane & ~3) | r);
          yr[r] = __shfl_sync(0xffffffffu, y0, (lane & ~3) | r);
        }
        sm::f2 acc[4][4];
        uint32_t a[2][2][4];
        {  // layer 0 (2 -> 32) on the FMA pipe, directly in accumulator layout
          const ulonglong2 wx01 = *reinterpret_cast<const ulonglong2*>(vq + 32 * sm::V_W0X), wx23 = *reinterpret_cast<const ulonglong2*>(vq + 32 * sm::V_W0X + 4);
          const ulonglong2 wy01 = *reinterpret_cast<const ulonglong2*>(vq + 32 * sm::V_W0Y), wy23 = *reinterpret_cast<const ulonglong2*>(vq + 32 * sm::V_W0Y + 4);
          const ulonglong2 b01 = *reinterpret_cast<const ulonglong2*>(vq + 32 * sm::V_B0), b23 = *reinterpret_cast<const ulonglong2*>(vq + 32 * sm::V_B0 + 4);
          const sm::f2 wx[4] = {wx01.x, wx01.y, wx23.x, wx23.y}, wy[4] = {wy01.x, wy01.y, wy23.x, wy23.y}, bb[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const sm::f2 x2 = tc::pk(xr[r], xr[r]), y2 = tc::pk(yr[r], yr[r]);
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[r][j] = tc::fma2(wy[j], y2, tc::fma2(wx[j], x2, bb[j]));
          }
        }
        sm::ln_tanh_frag(acc, vq + 32 * sm::V_G1, vq + 32 * sm::V_BE1, lane, a);
        sm::dense_frag<4>(wl + 0 * 128, bqq + 16 * 0, a, acc);
        sm::relu_frag(acc, a);
        sm::dense_frag<4>(wl + 1 * 128, bqq + 16 * 1, a, acc);
        sm::ln_tanh_frag(acc, vq + 32 * sm::V_G6, vq + 32 * sm::V_BE6, lane, a);
        sm::dense_frag<4>(wl + 2 * 128, bqq + 16 * 2, a, acc);
        sm::relu_frag(acc, a);
        sm::dense_frag<4>(wl + 3 * 128, bqq + 16 * 3, a, acc);
        sm::ln_tanh_frag(acc, vq + 32 * sm::V_G11, vq + 32 * sm::V_BE11, lane, a);
        sm::f2 mu[4][1];
        sm::dense_frag<1>(wl + 4 * 128, bqq + 16 * 4, a, mu);

        // head: d~ = relu(mu)^T (G p0 - h): partial over the lane's two channels for each row slot, transposing quad reduction
        float dp[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          float m0, m1;
          tc::upk(mu[r][0], m0, m1);
          const float ge0 = fmaf(gy0, yr[r], gx0 * xr[r]) - h0, ge1 = fmaf(gy1, yr[r], gx1 * xr[r]) - h1;
          dp[r] = fmaf(fmaxf(m1, 0.f), ge1, fmaxf(m0, 0.f) * ge0);
        }
        const float dn = sm::quad_transpose_sum(dp, tq);  // the lane's own point
        if (!hit) {
          float sa = 0.f;
#pragma unroll
          for (int e = 0; e < kMaxEdges; ++e)
            if (e < E) sa += fabsf(fmaf(prm.geo.G[e][1], y0, prm.geo.G[e][0] * x0) - prm.geo.h[e]);
          d = dn;
          eps = fmaf(prm.c_mu, sa, 1e-4f);
        }
      }
#pragma unroll
      for (int j = kP - 1; j > 0; --j) { kk[j] = kk[j - 1]; ll[j] = ll[j - 1]; dd[j] = dd[j - 1]; }
      kk[0] = i < n ? unique_key(orderable(d + eps), i) : 0xFFFFFFFFu;
      ll[0] = d - eps; dd[0] = d;
    }
    if (item + (int)gridDim.x < items) {  // this thread is done with `raw`: its part of the next item
      if (stage_points(item + (int)gridDim.x)) staged = item + (int)gridDim.x;
    }
    if (NB_WHATIF & 4) {
      if (tid == 0) prm.cand_cnt[item] = (kk[0] ^ kk[kP - 1]) == 12345u ? (int)(ll[0] + ll[kP - 1] + dd[0] + dd[kP - 1]) : 0;
      continue;
    }
    if (n <= kCandMax) {  // calibration mode: all points (they belong to warp 0's only tile), with their screened distance
      if (kk[0] != 0xFFFFFFFFu) { out_idx[kk[0] & kIdxMask] = (int)(kk[0] & kIdxMask); out_dt[kk[0] & kIdxMask] = dd[0]; }
      if (tid == 0) { prm.cand_cnt[item] = n; tc::refine_append(prm, item, n); }
      continue;
    }
    // ---- tau = the M-th smallest upper bound: unique 32-bit keys, M REDUX rounds per warp (each removes the one entry that equals
    // the minimum), then every warp merges the 4 M survivors the same way.  Two block barriers per item: the per-warp lists, and
    // the candidate list; the candidate counter alternates between two words so that resetting it needs no third one.
    {
      uint32_t q[kP];
#pragma unroll
      for (int j = 0; j < kP; ++j) q[j] = kk[j];
      for (int m = 0; m < M; ++m) {
        uint32_t mine = q[0];
#pragma unroll
        for (int j = 1; j < kP; ++j) mine = min(mine, q[j]);
        const uint32_t md = __reduce_min_sync(0xffffffffu, mine);
#pragma unroll
        for (int j = 0; j < kP; ++j) q[j] = q[j] == md ? 0xFFFFFFFFu : q[j];
        if (lane == 0) c32[warp * M + m] = md;
      }
    }
    __syncthreads();
    uint32_t tau = 0xFFFFFFFFu;
    {
      const int nc4 = 4 * M;  // <= 128 (M <= 32)
      uint32_t q0 = lane < nc4 ? c32[lane] : 0xFFFFFFFFu;
      uint32_t q1 = lane + 32 < nc4 ? c32[lane + 32] : 0xFFFFFFFFu;
      uint32_t q2 = lane + 64 < nc4 ? c32[lane + 64] : 0xFFFFFFFFu;
      uint32_t q3 = lane + 96 < nc4 ? c32[lane + 96] : 0xFFFFFFFFu;
      for (int m = 0; m < M; ++m) {  // n > kCandMax >= M: M finite keys exist
        tau = __reduce_min_sync(0xffffffffu, min(min(q0, q1), min(q2, q3)));
        q0 = q0 == tau ? 0xFFFFFFFFu : q0; q1 = q1 == tau ? 0xFFFFFFFFu : q1;
        q2 = q2 == tau ? 0xFFFFFFFFu : q2; q3 = q3 == tau ? 0xFFFFFFFFu : q3;
      }
    }
    auto take = [&](uint32_t k, float lb, float dt) {
      if (k != 0xFFFFFFFFu && orderable(lb) <= tau) {
        const int pos = atomicAdd(&cnt_s[par], 1);
        if (pos < kCandMax) { list_s[pos] = (int)(k & kIdxMask); ldt_s[pos] = dt; lrad_s[pos] = dt - lb; }
      }
    };
#pragma unroll
    for (int j = 0; j < kP; ++j) take(kk[j], ll[j], dd[j]);
    __syncthreads();
    const int nc = cnt_s[par];
    if (nc <= kCandMax) {
      if (tid < nc) { out_idx[tid] = list_s[tid]; out_dt[tid] = ldt_s[tid]; prm.cand_rad[(size_t)item * kCandMax + tid] = lrad_s[tid]; }
      if (tid == 0) {
        prm.cand_cnt[item] = nc;
        tc::refine_append(prm, item, nc);
        atomicAdd(&prm.screen_stats[2], (unsigned)nc);
        atomicAdd(&prm.screen_stats[3], 1u);
      }
    } else if (tid == 0) {
      prm.cand_cnt[item] = -1;  // too many candidates: the exact kernel evaluates this item in full
      atomicAdd(&prm.screen_stats[1], 1u);
      prm.flag_list[atomicAdd(prm.flag_count, 1)] = item;
    }
    // every thread has passed this item's first barrier, hence finished reading the OTHER counter (the previous item's) long ago
    if (tid == 0) cnt_s[par ^ 1] = 0;
    par ^= 1;
  }
  tc::cp_async_wait_all();
}

// ---- Clouds of <= 512 points: one warp per (environment, step) item.
// The T+1 items of an environment share its cloud, so a CTA of kScreenWarps warps is persistent over ENVIRONMENTS (over `parts` CTAs
// per environment when the batch is smaller than the resident grid, each with every parts-th group of W items): the cloud (x | y |
// vx | vy) is staged once per environment by cp.async, double-buffered (the next environment's copy is issued right after the barrier
// that opens the current one: one block barrier per environment).  The warps take the environment's items one at a time; lane l of a
// warp computes the frame of the warp's l-th item (one sincos per step) and the item loop broadcasts it by shuffle.  Per item, a lane
// owns point 32 j + 8 tq + g of every 32-point tile j (the row slot layout of the network, see the top of this file): all table
// gathers of the item are issued before any is consumed; a tile with a point outside the table (every tile when there is no table)
// then runs the network.  tau = the M-th smallest key of the warp (M REDUX rounds), the candidates are compacted by ballot: no merge
// stage, no block barrier, no shared-memory atomics per item.  Candidate and item counts, and the refine lists, are collected in
// shared memory and reach global memory once per environment (refine lists: one atomic per size class) or once per CTA (statistics).
//
// Two-level table path.  Of the ~500 points of an item only about M become candidates, so an item whose points all lie in the table
// first bounds every point from the coarse bound table (dune_table_coarse_kernel: one 4-byte load per point from a ~11 KB table that
// stays in L1, no fine-table gather) and gathers the fine cell only for the points that survive:
//   coarse pass: key_c = unique_key(orderable(UB_c), i); tau_c = the M-th smallest key_c (M REDUX rounds, as below);
//   survivors:   orderable(LB_c) <= tau_c, compacted by ballot in (tile j, lane) order (at most kSurvMax, 2 per lane);
//   fine pass:   the fine bounds of the survivors with the one-level path's arithmetic; tau_f = the M-th smallest fine key among them;
//                candidates: the survivors with orderable(d - rad) <= tau_f, written in survivor order.
// Why the candidates are the one-level path's, bit for bit (LB_f, UB_f: a point's fine bounds fl(d - rad), fl(d + rad); tau: the
// one-level path's M-th smallest fine key over all points):
//   - LB_c <= LB_f and UB_c >= UB_f at every point, and unique_key is monotone, so key_c >= key_f point by point and tau_c >= tau.
//   - A culled point has orderable(LB_f) >= orderable(LB_c) > tau_c >= tau: the one-level path rejects it as well.
//   - A point with key_f <= tau has orderable(LB_c) <= orderable(LB_f) <= orderable(UB_f) < key_f <= tau <= tau_c (unique_key rounds
//     up past the low 9 bits), so it survives: the M smallest fine keys are all survivors' and tau_f = tau.
//   - So survivors and one-level path take the same candidates, and the survivor order is the one-level order restricted to them.
// cand_idx / cand_dt / cand_rad / cand_cnt, the refine lists and the statistics are therefore those of the one-level path.  An item
// with a point outside the table (NaN included) or more than kSurvMax survivors takes the one-level path, as does every item when
// the handle has no coarse table (NB_SCREEN_COARSE=0).
constexpr int kWarpTiles = 16;  // 32-point tiles of an item: N <= 512, 9 index bits in the key (tc::unique_key)
// warps per CTA and CTAs per SM the register allocation is made for (128 registers).  Measured on C4 (H100 80GB HBM3, 700 W, bench.py
// 10 steps, 3 runs each): 4 warps x 4 CTAs 16.27-16.41 ms per step, 5 x 3 16.54-16.59 ms, 8 x 2 16.61-16.64 ms.
#ifndef NB_SCREEN_WARPS
#define NB_SCREEN_WARPS 4
#endif
#ifndef NB_SCREEN_WARP_BLOCKS
#define NB_SCREEN_WARP_BLOCKS 4
#endif
constexpr int kScreenWarps = NB_SCREEN_WARPS;
#ifndef NB_SCREEN_GATHER
#define NB_SCREEN_GATHER 4
#endif
constexpr int kGather = NB_SCREEN_GATHER;  // table gathers in flight per lane
constexpr int kSurvMax = 64;  // survivors of the coarse pass the two-level path holds: two per lane, their indices in the warp's net area

// shared memory: B fragments | permuted vectors | bias fragments | two clouds (x | y | vx | vy, N floats each) | per-warp network
// results (kWarpTiles x 32 float2) | refine lists of two environments ([parity][size class][T+1] items)
__host__ __device__ inline size_t dune_screen_warp_smem_bytes(int N, int T) {
  return (size_t)sm::kFragBytes + sm::kVecBytes + sm::kBiasQBytes + (size_t)2 * 4 * N * 4 + (size_t)kScreenWarps * kWarpTiles * 32 * 8 +
         (size_t)2 * 2 * (T + 1) * 4;
}

__global__ void __launch_bounds__(32 * kScreenWarps, NB_SCREEN_WARP_BLOCKS)
    dune_screen_warp_kernel(const DuneParams prm, const unsigned char* __restrict__ image, int parts) {
  constexpr int W = kScreenWarps, kThreads = 32 * W;
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  uint4* wfrag = reinterpret_cast<uint4*>(smem_dyn);
  float* vec = reinterpret_cast<float*>(smem_dyn + sm::kFragBytes);
  float4* biasq = reinterpret_cast<float4*>(smem_dyn + sm::kFragBytes + sm::kVecBytes);
  float* cloud = reinterpret_cast<float*>(smem_dyn + sm::kFragBytes + sm::kVecBytes + sm::kBiasQBytes);
  const int T1 = prm.T + 1, N = prm.N, M = prm.M, B = prm.B;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, tq = lane & 3;
  float2* net = reinterpret_cast<float2*>(cloud + (size_t)8 * N) + (size_t)warp * kWarpTiles * 32;
  int* rlist = reinterpret_cast<int*>(cloud + (size_t)8 * N + (size_t)W * kWarpTiles * 64);
  __shared__ int rcnt_s[2][2];   // [parity][size class] lengths of the refine lists in rlist
  __shared__ unsigned stat_s[4];  // candidates and items screened by this CTA (screen_stats[2], [3]), coarse survivors and items of the
                                 // one-level table path (coarse_stats[0], [1])
  __shared__ float4 frame_s[W][32];  // per warp: {sx, sy, cos, sin} of the steps of its next <= 32 items

  sm::stage_operands(image, wfrag, vec, biasq, tid, kThreads);
  if (tid < 4) rcnt_s[tid >> 1][tid & 1] = 0;
  if (tid < 4) stat_s[tid] = 0;
  const uint4* wl = wfrag + lane;
  const float* vq = vec + 8 * tq;
  const float4* bqq = biasq + 4 * tq;
  const int own = 8 * tq + g;  // the lane's point in every tile
  const int t_first = prm.skip_t0 ? 1 : 0;

  // the points of environment bb its items screen (0: none -- inactive, or <= 32 points outside calibration: every point is a candidate)
  auto screened_points = [&](int bb) -> int {
    if (prm.active && prm.active[bb] == 0) return 0;
    int nn = prm.num_points ? prm.num_points[bb] : N;
    nn = nn > N ? N : nn;
    return nn <= 0 || (nn <= kCandMax && !prm.calibrate) ? 0 : nn;
  };
  auto stage_cloud = [&](int bb, float* dst) {
    const int nn = screened_points(bb);
    const float* px = prm.points + (size_t)bb * 2 * N;
    const float* vx = prm.velocities ? prm.velocities + (size_t)bb * 2 * N : nullptr;
    for (int i = tid; i < nn; i += kThreads) {
      tc::cp_async4(dst + i, px + i);
      tc::cp_async4(dst + N + i, px + N + i);
      if (vx) {
        tc::cp_async4(dst + 2 * N + i, vx + i);
        tc::cp_async4(dst + 3 * N + i, vx + N + i);
      }
    }
  };
  // lane 0: item -> the refine list of its size class, in shared memory (dune_refine_kernel packs two items of <= 16 candidates into one warp)
  auto refine_push = [&](int par, int item, int nc) {
    if (nc <= 0) return;
    const int big = nc > 16 ? 1 : 0;
    rlist[(par * 2 + big) * T1 + atomicAdd(&rcnt_s[par][big], 1)] = item;
  };
  // one warp: the refine lists of parity par to global memory, one atomic per non-empty size class
  auto refine_flush = [&](int par) {
#pragma unroll 1
    for (int big = 0; big < 2; ++big) {
      const int c = rcnt_s[par][big];
      if (c == 0) continue;
      int pos = 0;
      if (lane == 0) pos = atomicAdd(prm.flag_count + 1 + big, c);
      pos = __shfl_sync(0xffffffffu, pos, 0);
      for (int x = lane; x < c; x += 32) prm.refine_list[(size_t)big * B * T1 + pos + x] = rlist[(par * 2 + big) * T1 + x];
      __syncwarp();
      if (lane == 0) rcnt_s[par][big] = 0;
    }
  };

  // work unit u = part u % parts of environment u / parts: its warp w takes the items t_first + (u % parts) W + w + k parts W
  const int units = B * parts, stride = parts * W;
  if ((int)blockIdx.x < units) stage_cloud(blockIdx.x / parts, cloud);
  int par = 0;  // parity of the CTA's unit: its cloud buffer and refine lists
  for (int u = blockIdx.x; u < units; u += gridDim.x, par ^= 1) {
    const int b = u / parts, part = u - b * parts;
    const float* raw = cloud + (size_t)par * 4 * N;
    tc::cp_async_wait_all();
    // environment b's cloud has landed for every thread; every warp is done with the previous unit (the other buffer and lists)
    __syncthreads();
    if (u + (int)gridDim.x < units) stage_cloud((u + gridDim.x) / parts, cloud + (size_t)(par ^ 1) * 4 * N);
    if (warp == W - 1) refine_flush(par ^ 1);

    const int act = prm.active ? prm.active[b] : 1;
    if (act == 0) {
      if (part == 0)
        for (int t = tid; t < T1; t += kThreads) prm.cand_cnt[(size_t)b * T1 + t] = 0;
      continue;
    }
    int n = prm.num_points ? prm.num_points[b] : N;
    n = n < 0 ? 0 : (n > N ? N : n);
    if (tid == 0 && part == 0) {
      if (prm.skip_t0) prm.cand_cnt[(size_t)b * T1] = 0;  // same inputs as in the previous PAN iteration: its outputs stand
      else {
        prm.sel_count[b] = n < M ? n : M;
        if (n == 0 && prm.min_dist) prm.min_dist[b] = __int_as_float(0x7f800000);
      }
    }
    const bool screen = n > kCandMax || prm.calibrate;
    const float* ns = prm.nom_s + (size_t)b * 3 * T1;

#pragma unroll 1
    for (int t0 = t_first + part * W + warp; t0 < T1; t0 += 32 * stride) {
      // lane l: the frame of this warp's item t0 + l stride (the arithmetic of tc::item_frame), read by every lane of the item
      __syncwarp();
      if (screen && t0 + lane * stride < T1) {
        const int tl = t0 + lane * stride;
        const float th = ns[2 * T1 + tl];
        frame_s[warp][lane] = make_float4(ns[tl], ns[T1 + tl], cosf(th), sinf(th));
      }
      __syncwarp();
#pragma unroll 1
      for (int l = 0; l < 32 && t0 + l * stride < T1; ++l) {
        const int t = t0 + l * stride, item = b * T1 + t;
        if (!screen) {  // nothing to screen: every point is a candidate
          if (lane < n) { prm.cand_idx[(size_t)item * kCandMax + lane] = lane; prm.cand_dt[(size_t)item * kCandMax + lane] = __int_as_float(0x7fc00000); }
          if (lane == 0) { prm.cand_cnt[item] = n; refine_push(par, item, n); }
          continue;
        }
        const float4 fr = frame_s[warp][l];
        const float sx = fr.x, sy = fr.y, cs = fr.z, sn = fr.w;
        // point i in the robot frame (tc::ItemFrame::local on the staged cloud); rows beyond n run on zeros (their results are never
        // looked at)
        auto local = [&](int i, float& x0, float& y0) {
          x0 = 0.f; y0 = 0.f;
          if (i < n) {
            float gx = raw[i], gy = raw[N + i];
            if (prm.velocities) {
              gx = flow(gx, raw[2 * N + i], prm.dt, t);
              gy = flow(gy, raw[3 * N + i], prm.dt, t);
            }
            const float dx = gx - sx, dy = gy - sy;
            x0 = fmaf(cs, dx, sn * dy);
            y0 = fmaf(cs, dy, -(sn * dx));
          }
        };

        const int tiles = (n + 31) >> 5;
        int32_t* out_idx = prm.cand_idx + (size_t)item * kCandMax;
        float* out_dt = prm.cand_dt + (size_t)item * kCandMax;
        const uint32_t below = (1u << lane) - 1u;
        // lane 0: the item's candidate count, refine list and statistics (nc <= kCandMax), or the item to the exact kernel
        auto finish = [&](int nc) {
          if (lane != 0) return;
          if (nc <= kCandMax) {
            prm.cand_cnt[item] = nc;
            refine_push(par, item, nc);
            atomicAdd(&stat_s[0], (unsigned)nc);
            atomicAdd(&stat_s[1], 1u);
          } else {
            prm.cand_cnt[item] = -1;  // too many candidates: the exact kernel evaluates this item in full
            atomicAdd(&prm.screen_stats[1], 1u);
            prm.flag_list[atomicAdd(prm.flag_count, 1)] = item;
          }
        };
        // candidate p: point i with screened distance d and error radius r
        auto put = [&](int p, int i, float d, float r) {
          const float lb = d - r;
          out_idx[p] = i;
          out_dt[p] = d;
          prm.cand_rad[(size_t)item * kCandMax + p] = d - lb;
        };
        if (prm.tab_coarse && n > kCandMax && NB_WHATIF == 0) {  // the two-level table path (see above the kernel)
          bool inside = true;
          uint32_t kc[kWarpTiles];
#pragma unroll
          for (int j = 0; j < kWarpTiles; ++j) {
            kc[j] = 0xFFFFFFFFu;
            const int i = 32 * j + own;
            if (j < tiles && i < n) {
              float x0, y0, a, bq;
              int ix, iy;
              local(i, x0, y0);
              if (table_cell_xy(prm, x0, y0, ix, iy, a, bq)) {
                const uint32_t lu = __ldg(prm.tab_coarse + (iy >> kCoarseLog) * prm.tab_cn + (ix >> kCoarseLog));
                net[32 * j + lane].x = __half2float(__ushort_as_half((unsigned short)(lu & 0xFFFFu)));
                kc[j] = tc::unique_key(orderable(__half2float(__ushort_as_half((unsigned short)(lu >> 16)))), i);
              } else {
                inside = false;
              }
            }
          }
          if (__all_sync(0xffffffffu, inside)) {
            uint32_t tau = 0u;
#pragma unroll 1
            for (int m = 0; m < M; ++m) {
              uint32_t mine = 0xFFFFFFFFu;
#pragma unroll
              for (int j = 0; j < kWarpTiles; ++j) mine = min(mine, kc[j] > tau ? kc[j] : 0xFFFFFFFFu);
              tau = __reduce_min_sync(0xffffffffu, mine);
            }
            uint32_t survm = 0u;
#pragma unroll
            for (int j = 0; j < kWarpTiles; ++j)
              if (kc[j] != 0xFFFFFFFFu && orderable(net[32 * j + lane].x) <= tau) survm |= 1u << j;
            __syncwarp();  // every lane has read its coarse bounds: the survivor list overwrites the start of the warp's net area
            int* surv = reinterpret_cast<int*>(net);
            int ns = 0;
#pragma unroll
            for (int j = 0; j < kWarpTiles; ++j) {
              const bool sv = (survm >> j) & 1u;
              const uint32_t bal = __ballot_sync(0xffffffffu, sv);
              const int p = ns + __popc(bal & below);
              if (sv && p < kSurvMax) surv[p] = 32 * j + own;
              ns += __popc(bal);
            }
            if (ns <= kSurvMax) {
              __syncwarp();
              int si[2];
              float4 cell[2];
              float rad[2], ca[2], cb[2];
#pragma unroll
              for (int r = 0; r < 2; ++r) {
                const int p = 32 * r + lane;
                si[r] = p < ns ? surv[p] : -1;
                int c = 0;
                ca[r] = 0.f; cb[r] = 0.f;
                if (si[r] >= 0) {
                  float x0, y0;
                  local(si[r], x0, y0);
                  table_cell(prm, x0, y0, c, ca[r], cb[r]);
                }
                cell[r] = __ldg(prm.tab_cell + c);
                rad[r] = __ldg(prm.tab_rad + c);
              }
              __syncwarp();  // the survivor list is read: the next item may write the net area
              float d[2];
              uint32_t kf[2];
#pragma unroll
              for (int r = 0; r < 2; ++r) {
                d[r] = table_bilerp(cell[r], ca[r], cb[r]);
                kf[r] = si[r] >= 0 ? tc::unique_key(orderable(d[r] + rad[r]), si[r]) : 0xFFFFFFFFu;
              }
              tau = 0u;
#pragma unroll 1
              for (int m = 0; m < M; ++m) {
                const uint32_t mine = min(kf[0] > tau ? kf[0] : 0xFFFFFFFFu, kf[1] > tau ? kf[1] : 0xFFFFFFFFu);
                tau = __reduce_min_sync(0xffffffffu, mine);
              }
              bool tk[2];
              int nc = 0;
#pragma unroll
              for (int r = 0; r < 2; ++r) {
                tk[r] = kf[r] != 0xFFFFFFFFu && orderable(d[r] - rad[r]) <= tau;
                nc += __popc(__ballot_sync(0xffffffffu, tk[r]));
              }
              if (nc <= kCandMax) {
                int pos = 0;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                  const uint32_t bal = __ballot_sync(0xffffffffu, tk[r]);
                  if (tk[r]) put(pos + __popc(bal & below), si[r], d[r], rad[r]);
                  pos += __popc(bal);
                }
              }
              finish(nc);
              if (lane == 0) atomicAdd(&stat_s[2], (unsigned)ns);
              continue;
            }
          }
          if (lane == 0) atomicAdd(&stat_s[3], 1u);
        }
        // one-level path: the bounds of the lane's points, d~ and its error radius, collect in net[32 j + lane] (tile j): from the table
        // where it covers the point, then from the network for the tiles with a point outside it (netm; every tile when there is no table)
        uint32_t netm = 0u;
        if (prm.tab_cell) {
          uint32_t hitm = 0u;  // bit j: the point of tile j lies in the table or beyond n
#pragma unroll 1
          for (int h = 0; h < tiles; h += kGather) {  // kGather tiles at a time: all their gathers are issued before any is consumed
            float4 cell[kGather];
            float rad[kGather], ca[kGather], cb[kGather];
#pragma unroll
            for (int q = 0; q < kGather; ++q) {
              const int j = h + q;
              if (j < tiles) {
                const int i = 32 * j + own;
                float x0, y0;
                local(i, x0, y0);
                int c = 0;  // a point outside the table, or beyond n, reads cell 0
                ca[q] = 0.f; cb[q] = 0.f;
                const bool hit = i >= n || table_cell(prm, x0, y0, c, ca[q], cb[q]);
                if (NB_WHATIF & 16) { c = 0; ca[q] = fabsf(x0) + fabsf(y0); }
                hitm |= hit ? 1u << j : 0u;
                if (!__all_sync(0xffffffffu, hit)) netm |= 1u << j;
                cell[q] = __ldg(prm.tab_cell + c);
                rad[q] = __ldg(prm.tab_rad + c);
              }
            }
#pragma unroll
            for (int q = 0; q < kGather; ++q)
              if (h + q < tiles)
                net[32 * (h + q) + lane] = (NB_WHATIF & 16) ? make_float2(ca[q] + 0.f * cell[q].x, fminf(rad[q], 0.05f))
                                                            : make_float2(table_bilerp(cell[q], ca[q], cb[q]), rad[q]);
          }
#pragma unroll 1
          for (uint32_t m = netm; m != 0u; m &= m - 1u) {
            const int j = __ffs(m) - 1, i = 32 * j + own;
            float x0, y0;
            local(i, x0, y0);
            const float dn = sm::tile_network(prm.geo, x0, y0, lane, wl, vq, bqq);
            if (!((hitm >> j) & 1u)) net[32 * j + lane] = make_float2(dn, sm::network_radius(prm, x0, y0));
          }
        } else {
#pragma unroll 1
          for (int j = 0; j < tiles; ++j) {
            const int i = 32 * j + own;
            float x0, y0;
            local(i, x0, y0);
            const float dn = sm::tile_network(prm.geo, x0, y0, lane, wl, vq, bqq);
            net[32 * j + lane] = make_float2(dn, sm::network_radius(prm, x0, y0));
          }
        }
        // upper-bound keys, unique through the point's index in the low 9 bits (the bounds stay in net)
        uint32_t key[kWarpTiles];
#pragma unroll
        for (int j = 0; j < kWarpTiles; ++j) {
          key[j] = 0xFFFFFFFFu;
          if (32 * j + own < n) {
            const float2 v = net[32 * j + lane];
            key[j] = tc::unique_key(orderable(v.x + v.y), 32 * j + own);
          }
        }
        if (NB_WHATIF & 4) {
          if (lane == 0) prm.cand_cnt[item] = (key[0] ^ key[kWarpTiles - 1]) == 12345u ? 1 : 0;
          continue;
        }
        if (n <= kCandMax) {  // calibration mode: all points (tile 0), with their screened distance
          if (key[0] != 0xFFFFFFFFu) { out_idx[own] = own; out_dt[own] = net[lane].x; }
          if (lane == 0) { prm.cand_cnt[item] = n; refine_push(par, item, n); }
          continue;
        }
        // tau = the M-th smallest upper bound: each REDUX round finds the smallest key above the previous one (keys are unique and
        // >= 0x200; n > kCandMax >= M: M finite keys exist)
        uint32_t tau = 0u;
#pragma unroll 1
        for (int m = 0; m < M; ++m) {
          uint32_t mine = 0xFFFFFFFFu;
#pragma unroll
          for (int j = 0; j < kWarpTiles; ++j) mine = min(mine, key[j] > tau ? key[j] : 0xFFFFFFFFu);
          tau = __reduce_min_sync(0xffffffffu, mine);
        }
        // the candidates: lower bound <= tau
        uint32_t takem = 0u;
        int nc = 0;
#pragma unroll
        for (int j = 0; j < kWarpTiles; ++j) {
          bool tk = false;
          if (key[j] != 0xFFFFFFFFu) {
            const float2 v = net[32 * j + lane];
            tk = orderable(v.x - v.y) <= tau;
          }
          takem |= tk ? 1u << j : 0u;
          nc += __popc(__ballot_sync(0xffffffffu, tk));
        }
        if (nc <= kCandMax) {
          int pos = 0;
#pragma unroll
          for (int j = 0; j < kWarpTiles; ++j) {
            const bool tk = (takem >> j) & 1u;
            const uint32_t bal = __ballot_sync(0xffffffffu, tk);
            if (tk) {
              const float2 v = net[32 * j + lane];
              put(pos + __popc(bal & below), 32 * j + own, v.x, v.y);
            }
            pos += __popc(bal);
          }
        }
        finish(nc);
      }
    }
  }
  tc::cp_async_wait_all();
  __syncthreads();
  if (warp == W - 1) {
    refine_flush(0);
    refine_flush(1);
  }
  if (tid == 0 && stat_s[1]) {
    atomicAdd(&prm.screen_stats[2], stat_s[0]);
    atomicAdd(&prm.screen_stats[3], stat_s[1]);
  }
  if (tid == 0 && (stat_s[2] || stat_s[3])) {
    atomicAdd(&prm.coarse_stats[0], stat_s[2]);
    atomicAdd(&prm.coarse_stats[1], stat_s[3]);
  }
}

}  // namespace nb
