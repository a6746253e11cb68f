// DUNE kernels, warpgroup versions (Hopper wgmma: B operand from shared memory, accumulators in registers).
//
// Point flow -> robot frame -> ObsPointNet -> distance -> M closest points (dune_common.cuh).
// Mapping: CTA = 128 threads = one warpgroup; thread r owns point r of a 128-point tile for the whole network, so LayerNorm
// statistics, tanh, ReLU and the distance are thread-local (no shuffles, no fragment bookkeeping).  Per dense layer:
//   registers --split x = hi + lo (fp16)--> shared-memory tile (A operand, canonical K-major layout)   [all threads]
//   D[128 x 32] = ONES.BIASB + A_lo.B_hi + A_hi.B_lo + A_hi.B_hi                                    [the warpgroup, wgmma
//                                                      m64n32k16 per 64-row half, B and ONES from shared memory]
//   accumulator fragments -> the same tile -> 32 fp32 columns = the thread's row                      [all threads]
//
// dune_tcp_kernel: two 128-point tiles ("slots") per CTA, each with its own 16 KB tile, interleaved by the same 128 threads.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "dune_common.cuh"  // DuneParams, orderable(), flow()

namespace nb {

// Weight image built on the host (dune_tc.cu): canonical K-major / no-swizzle wgmma operand layout
// (core matrix = 8 rows x 16 B; SBO = 128 B between 8-row groups; LBO between the two 8-half K groups).
struct TcImage {
  static constexpr int kLayerStride = 4096;  // per dense layer (4 hidden + head, all N = 32): W_hi 2048 | W_lo 2048
  static constexpr int kLayers = 5;          // the head's rows E..31 are zero
  static constexpr int kFloatOff = kLayers * kLayerStride;  // 20480
  // float section (offsets in floats): W0 (32x2, row-major), b0, LayerNorm gain/offset pre-multiplied by 2*log2(e),
  // the biases of the five dense layers (already including the folded tanh map; head zero padded to 32), and W0
  // again as two columns (W0X[j] = W0[j][0], W0Y[j] = W0[j][1]) for the layer-0 loop
  static constexpr int W0 = 0, B0 = 64, G1 = 96, BE1 = 128, G6 = 160, BE6 = 192, G11 = 224, BE11 = 256, BH = 288, W0X = 448, W0Y = 480,
                       kFloats = 512;
  // bias by tensor core: D = ONES[128 x 16] . BIASB[layer][32 x 16] with ONES(m, 0..2) = 1 and BIASB(n, 0..2) = the three
  // fp16 pieces of the bias (hi, lo, lo2) -- the first MMA of a layer, so that the accumulators need no initialisation from
  // shared memory.  Both are K-major / no-swizzle core-matrix images like the weights.
  static constexpr int kOnesOff = kFloatOff + kFloats * 4;   // 22528, 4096 B  (LBO 2048)
  static constexpr int kBiasBOff = kOnesOff + 4096;          // 26624, 5 x 1024 B (LBO 512)
  static constexpr int kBytes = kBiasBOff + kLayers * 1024;  // 31744 (a multiple of 1024: the tiles that follow stay aligned)
};

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- the 128-row tile ------------------------------------------------------------------------------------------------
// A operand of a layer: 128 rows x 32 K, fp16 hi at bytes [0, 8192), lo at [8192, 16384), each in the canonical K-major /
// no-swizzle layout (row p, K group q of 8 halves at q * 2048 + p * 16: LBO 2048, SBO 128, 4096 B per K step of 16).
// Once the layer's MMAs have completed, the same 16 KB hold its fp32 output D: features 4c..4c+3 of row p lie in the
// 16 bytes of A's chunk c (c = 0..7) of the same row, so every row's output replaces exactly that row's operands.
constexpr int kTileBytes = 16384;
__device__ __forceinline__ int chunk_off(int p, int c) { return c * 2048 + p * 16; }

// Row of the tile that thread r of the warpgroup owns.  wgmma gives warp w the accumulators of rows 16w..16w+15 of each
// 64-row half; placing lanes 0-15 of warp w in the first half and lanes 16-31 in the second makes the warp's accumulators
// exactly its own 32 rows, so D reaches its owners through shared memory with a warp barrier only.
__device__ __forceinline__ int tile_row(int r) { return ((r & 16) << 2) | ((r >> 5) << 4) | (r & 15); }

// the thread's activations (K 0..31 as 16 fp16 pairs, hi and lo) -> its row of the A operand
__device__ __forceinline__ void st_a(unsigned char* tile, int p, const uint32_t (&hi)[16], const uint32_t (&lo)[16]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    *reinterpret_cast<uint4*>(tile + chunk_off(p, q)) = make_uint4(hi[4 * q], hi[4 * q + 1], hi[4 * q + 2], hi[4 * q + 3]);
    *reinterpret_cast<uint4*>(tile + chunk_off(p, 4 + q)) = make_uint4(lo[4 * q], lo[4 * q + 1], lo[4 * q + 2], lo[4 * q + 3]);
  }
}

// wgmma shared-memory descriptor, no swizzle: start address, LBO, SBO = 128 B (all operands lie in the first 256 KB)
__device__ __forceinline__ uint64_t desc(uint32_t saddr, uint32_t lbo_bytes) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(128u >> 4) << 32);
}

// D[64 x 32] += A[64 x 16] . B[32 x 16]^T, fp16 operands, fp32 accumulators
__device__ __forceinline__ void wgmma32(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
        "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db)
      : "memory");
}

// D[64 x 32] = A[64 x 16] . B[32 x 16]^T (scale-d = 0: D is written, not read)
__device__ __forceinline__ void wgmma32_first(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, 0, 1, 1, 0, 0;"
      : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]), "=f"(d[9]), "=f"(d[10]),
        "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15])
      : "l"(da), "l"(db)
      : "memory");
}

// One dense layer of the tile, issued by the 128 threads of a warpgroup after a barrier that made every row of A visible
// to the async proxy (st_a + fence.proxy.async + barrier):
//   kLo = true:  D = ONES.BIASB[layer] + A_lo.B_hi + A_hi.B_lo + A_hi.B_hi   (3-pass fp16 split, fp32 accuracy)
//   kLo = false: D = ONES.BIASB[layer] + A_hi.B_hi                           (single pass: the screening network)
// then D replaces A in the tile.  `img` is the shared-memory address of the operand image.
template <bool kLo>
__device__ __forceinline__ void layer_mma(unsigned char* tile, uint32_t img, int layer, int warp, int lane) {
  using I = TcImage;
  const uint32_t ta = smem_u32(tile);
  float d[2][16];
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
  const uint64_t ones = desc(img + I::kOnesOff, 2048), biasb = desc(img + I::kBiasBOff + layer * 1024, 512);
  const uint32_t w = img + layer * I::kLayerStride;
#pragma unroll
  for (int h = 0; h < 2; ++h) {  // rows 64 h .. 64 h + 63: 8 row groups of 128 B further
    const uint32_t a = ta + h * 1024;
    wgmma32_first(d[h], ones, biasb);
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const uint64_t bhi = desc(w + s * 1024, 512), ahi = desc(a + s * 4096, 2048);
      if (kLo) {
        wgmma32(d[h], desc(a + 8192 + s * 4096, 2048), bhi);  // A_lo . B_hi (small terms first)
        wgmma32(d[h], ahi, desc(w + 2048 + s * 1024, 512));   // A_hi . B_lo
      }
      wgmma32(d[h], ahi, bhi);  // A_hi . B_hi
    }
  }
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
  asm volatile("bar.sync 1, 128;" ::: "memory");  // every warp's MMAs have read A before any D overwrites it
  // accumulator i of half h: row 16 warp + g + 8 ((i >> 1) & 1) of the half, column 8 (i >> 2) + 2 tq + (i & 1)
  const int g = lane >> 2, tq = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 16; i += 2) {
      const int p = 64 * h + 16 * warp + g + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * tq;
      *reinterpret_cast<float2*>(tile + chunk_off(p, col >> 2) + (col & 3) * 4) = make_float2(d[h][i], d[h][i + 1]);
    }
  __syncwarp();
}

// ---- packed pairs of FP32 values (two features per 64-bit register pair, low word = even feature) ----------------------
// Each operation is two correctly rounded scalar operations; the explicit _rn intrinsics keep the compiler from contracting
// a multiply and an add into one FMA, so every result has the bits the formula states.
using f2 = unsigned long long;
__device__ __forceinline__ f2 pk(float lo, float hi) { f2 r; asm("mov.b64 %0, {%1,%2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ f2 pku(uint32_t lo, uint32_t hi) { f2 r; asm("mov.b64 %0, {%1,%2};" : "=l"(r) : "r"(lo), "r"(hi)); return r; }
__device__ __forceinline__ void upk(f2 v, float& lo, float& hi) { asm("mov.b64 {%0,%1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) {
  float a0, a1, b0, b1, c0, c1;
  upk(a, a0, a1); upk(b, b0, b1); upk(c, c0, c1);
  return pk(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ f2 add2(f2 a, f2 b) {
  float a0, a1, b0, b1;
  upk(a, a0, a1); upk(b, b0, b1);
  return pk(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ f2 mul2(f2 a, f2 b) {
  float a0, a1, b0, b1;
  upk(a, a0, a1); upk(b, b0, b1);
  return pk(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}

// the thread's row of D (32 fp32 features) as 16 pairs / the first 8 features (the head)
__device__ __forceinline__ void ld32p(const unsigned char* tile, int p, f2 (&hp)[16]) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const uint4 v = *reinterpret_cast<const uint4*>(tile + chunk_off(p, c));
    hp[2 * c] = pku(v.x, v.y);
    hp[2 * c + 1] = pku(v.z, v.w);
  }
}
__device__ __forceinline__ void ld8(const unsigned char* tile, int p, float (&h)[8]) {
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const float4 v = *reinterpret_cast<const float4*>(tile + chunk_off(p, c));
    h[4 * c] = v.x; h[4 * c + 1] = v.y; h[4 * c + 2] = v.z; h[4 * c + 3] = v.w;
  }
}

// (a0, a1) -> hi = fp16x2(a), lo = fp16x2(a - hi)  (a - hi is exact to one rounding, like a fused a + hi * -1)
__device__ __forceinline__ void split_pair(float a0, float a1, uint32_t& hi, uint32_t& lo) {
  const __half2 hh = __floats2half2_rn(a0, a1);
  hi = *reinterpret_cast<const uint32_t*>(&hh);
  const float2 f = __half22float2(hh);
  const __half2 ll = __floats2half2_rn(__fsub_rn(a0, f.x), __fsub_rn(a1, f.y));
  lo = *reinterpret_cast<const uint32_t*>(&ll);
}

// LayerNorm (eps 1e-5, biased variance) + r = 1/(exp2(.)+1) + fp16 split.  The inputs arrive CENTRED: the layer that
// produces them has W - colmean(W), b - mean(b) (host image), so mean(h) = 0 up to rounding and only the variance is left.
// tanh(y) = 1 - 2r with r = 1/(exp2(a) + 1), a = 2*log2(e)*y; the affine map 1 - 2r is folded into the weights and bias of
// the layer that follows (W' = -2W, b' = b + rowsum(W), built on the host), so r itself is the activation.
// kFast: one MUFU.RCP serves four features: with d_i = exp2(a_i) + 1,  t = 1/(d0 d1 d2 d3),  1/d0 = t d1 d2 d3, ...  (the
// host enables it only if the checkpoint's LayerNorm gains/offsets bound every a_i by 30, so that the product of four stays
// below 2^124)
template <bool kFast>
__device__ __forceinline__ void ln_tanh_split(f2 (&hp)[16], const float* __restrict__ g, const float* __restrict__ be, uint32_t (&hi)[16],
                                              uint32_t (&lo)[16]) {
  f2 qa = 0ull, qb = 0ull, qc = 0ull, qd = 0ull;
#pragma unroll
  for (int c = 0; c < 16; c += 4) {
    qa = fma2(hp[c], hp[c], qa);
    qb = fma2(hp[c + 1], hp[c + 1], qb);
    qc = fma2(hp[c + 2], hp[c + 2], qc);
    qd = fma2(hp[c + 3], hp[c + 3], qd);
  }
  float q0, q1;
  upk(add2(add2(qa, qb), add2(qc, qd)), q0, q1);
  float r;  // the argument is >= 1e-5: no denormal guard needed
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(fmaf(q0 + q1, 1.0f / 32, 1e-5f)));
  const f2 r2 = pk(r, r), one2 = pk(1.0f, 1.0f);
#pragma unroll
  for (int c = 0; c < 16; c += 2) {
    const ulonglong2 gg = *reinterpret_cast<const ulonglong2*>(g + 2 * c);
    const ulonglong2 bb = *reinterpret_cast<const ulonglong2*>(be + 2 * c);
    float a0, a1, a2, a3, e0, e1, e2, e3;
    upk(fma2(mul2(hp[c], r2), gg.x, bb.x), a0, a1);
    upk(fma2(mul2(hp[c + 1], r2), gg.y, bb.y), a2, a3);
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(a0));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(a1));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e2) : "f"(a2));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e3) : "f"(a3));
    const f2 da = add2(pk(e0, e1), one2), db = add2(pk(e2, e3), one2);  // (d0, d1), (d2, d3)
    float r0, r1, r2s, r3;
    if (kFast) {
      float p0, p1, t;
      upk(mul2(da, db), p0, p1);  // (d0 d2, d1 d3)
      const float pp = p0 * p1;
      asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(pp));
      const f2 u = pk(t * p1, t * p0);  // (1/(d0 d2), 1/(d1 d3))
      upk(mul2(u, db), r0, r1);         // 1/d0, 1/d1
      upk(mul2(u, da), r2s, r3);        // 1/d2, 1/d3
    } else {
      float d0, d1, d2, d3;
      upk(da, d0, d1);
      upk(db, d2, d3);
      asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r0) : "f"(d0));
      asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r1) : "f"(d1));
      asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r2s) : "f"(d2));
      asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r3) : "f"(d3));
    }
    split_pair(r0, r1, hi[c], lo[c]);
    split_pair(r2s, r3, hi[c + 1], lo[c + 1]);
  }
}

// relu + split without a max: hi = fp16x2(relu(a)) rounded TOWARDS ZERO (cvt.rz.relu), so that a - hi is >= 0 for a > 0
// and equals a < 0 for a <= 0 (hi = 0); lo = fp16x2(relu(a - hi)) then drops exactly the negative inputs
__device__ __forceinline__ void relu_split(const f2 (&hp)[16], uint32_t (&hi)[16], uint32_t (&lo)[16]) {
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    float a0, a1;
    upk(hp[c], a0, a1);
    asm("cvt.rz.relu.f16x2.f32 %0, %1, %2;" : "=r"(hi[c]) : "f"(a1), "f"(a0));  // d = {hi half: first source, lo half: second}
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hi[c]));
    asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(lo[c]) : "f"(__fsub_rn(a1, f.y)), "f"(__fsub_rn(a0, f.x)));
  }
}

}  // namespace tc

// shared memory: operand image | two tiles | keys (N x 8 B, n > 512) | smu (N x E floats) | candidates (4 warps x M)
__host__ __device__ inline size_t dune_tc_smem_bytes(int N, int E, int M) {
  return TcImage::kBytes + 2 * (size_t)tc::kTileBytes + (size_t)N * 8 + (((size_t)N * E * 4 + 7) / 8) * 8 + (size_t)4 * M * 8 + 64;
}

namespace tc {

// point i of env b at step t in the robot frame of the nominal state: p0 = R^T (p_t - trans)   (pan.py:210)
struct ItemFrame {
  float sx, sy, cs, sn, dt;
  const float *px, *py, *vx, *vy;
  int t;
  __device__ __forceinline__ void world(int i, float& gx, float& gy) const {
    gx = px[i]; gy = py[i];
    if (vx) {
      gx = flow(gx, vx[i], dt, t);
      gy = flow(gy, vy[i], dt, t);
    }
  }
  __device__ __forceinline__ void local(int i, float& x0, float& y0) const {
    float gx, gy;
    world(i, gx, gy);
    const float dx = gx - sx, dy = gy - sy;
    x0 = fmaf(cs, dx, sn * dy);
    y0 = fmaf(cs, dy, -(sn * dx));
  }
};

__device__ __forceinline__ ItemFrame item_frame(const DuneParams& prm, int b, int t) {
  const int T1 = prm.T + 1;
  const float* ns = prm.nom_s + (size_t)b * 3 * T1;
  ItemFrame f;
  f.sx = ns[t]; f.sy = ns[T1 + t];
  const float th = ns[2 * T1 + t];
  f.cs = cosf(th); f.sn = sinf(th);
  f.dt = prm.dt; f.t = t;
  f.px = prm.points + (size_t)b * 2 * prm.N;
  f.py = f.px + prm.N;
  f.vx = prm.velocities ? prm.velocities + (size_t)b * 2 * prm.N : nullptr;
  f.vy = f.vx ? f.vx + prm.N : nullptr;
  return f;
}

// layer 0 (2 -> 32, FMA pipe) of the point (x0, y0), features `off` .. `off` + 2 cnt - 1 as pairs
template <int kPairs>
__device__ __forceinline__ void layer0(const float* __restrict__ fl, float x0, float y0, int off, f2 (&hp)[kPairs]) {
  using I = TcImage;
  const f2 x2 = pk(x0, x0), y2 = pk(y0, y0);
#pragma unroll
  for (int c = 0; c < kPairs; c += 2) {
    const ulonglong2 wx = *reinterpret_cast<const ulonglong2*>(fl + I::W0X + off + 2 * c);
    const ulonglong2 wy = *reinterpret_cast<const ulonglong2*>(fl + I::W0Y + off + 2 * c);
    const ulonglong2 bb = *reinterpret_cast<const ulonglong2*>(fl + I::B0 + off + 2 * c);
    hp[c] = fma2(wy.x, y2, fma2(wx.x, x2, bb.x));
    hp[c + 1] = fma2(wy.y, y2, fma2(wx.y, x2, bb.y));
  }
}

// mu = relu(head), dist = mu^T (G p0 - h)   (dune.py:119-122); publishes mu and the sortable key of the point
__device__ __forceinline__ uint32_t finish_point(const DuneParams& prm, float (&mu)[8], float x0, float y0, int i, bool valid, int E, float* smu,
                                                 unsigned long long* keys) {
  float d = 0.f;
#pragma unroll
  for (int e = 0; e < kMaxEdges; ++e) {
    if (e < E) {
      mu[e] = fmaxf(mu[e], 0.f);
      const float ge = fmaf(prm.geo.G[e][1], y0, prm.geo.G[e][0] * x0) - prm.geo.h[e];
      d = fmaf(mu[e], ge, d);
      if (valid) smu[i * E + e] = mu[e];
    }
  }
  const uint32_t key = orderable(d);
  if (valid && keys) keys[i] = ((unsigned long long)key << 32) | (unsigned)i;
  return valid ? key : 0xFFFFFFFFu;
}

// top-M (ascending, ties -> lower index) of the item's keys and the output rows; called by the 4 compute warps of a CTA
// after a block barrier that made keys / smu visible.  Contains one block barrier.
__device__ __forceinline__ void select_and_write(const DuneParams& prm, const ItemFrame& fr, int b, int t, int n, int cnt, int warp, int lane,
                                                 unsigned long long* keys, const float* smu, unsigned long long* cands) {
  const int M = prm.M, E = prm.geo.E, T1 = prm.T + 1;
  unsigned long long mine = ~0ull;
  {
    unsigned long long* cand = cands + warp * M;
    for (int m = 0; m < cnt; ++m) {  // per-warp REDUX rounds over the keys of the rows this warp computed
      unsigned bd = 0xFFFFFFFFu, bi = 0xFFFFFFFFu;
      for (int i = warp * 32 + lane; i < n; i += 128) {
        const uint2 k = *reinterpret_cast<const uint2*>(keys + i);
        if (k.y < bd) { bd = k.y; bi = k.x; }
      }
      const unsigned md = __reduce_min_sync(0xffffffffu, bd);
      const unsigned mi = __reduce_min_sync(0xffffffffu, bd == md ? bi : 0xFFFFFFFFu);
      if (md != 0xFFFFFFFFu && bd == md && bi == mi) keys[mi] = ~0ull;
      if (lane == 0) cand[m] = md == 0xFFFFFFFFu ? ~0ull : (((unsigned long long)md << 32) | mi);
      __syncwarp();
    }
  }
  __syncthreads();
  if (warp == 0) {  // merge the 4 candidate lists
    const int total = 4 * cnt;
    for (int m = 0; m < cnt; ++m) {
      unsigned bd = 0xFFFFFFFFu, bi = 0xFFFFFFFFu;
      int bpos = -1;
      for (int c = lane; c < total; c += 32) {
        const int w = c / cnt, r = c - w * cnt;
        const uint2 k = *reinterpret_cast<const uint2*>(cands + w * M + r);
        if (k.y < bd || (k.y == bd && k.x < bi)) { bd = k.y; bi = k.x; bpos = w * M + r; }
      }
      const unsigned md = __reduce_min_sync(0xffffffffu, bd);
      const unsigned mi = __reduce_min_sync(0xffffffffu, bd == md ? bi : 0xFFFFFFFFu);
      if (bpos >= 0 && bd == md && bi == mi) cands[bpos] = ~0ull;
      if (lane == m) mine = ((unsigned long long)md << 32) | mi;
      __syncwarp();
    }
    if (lane < cnt) {  // lane m writes the m-th closest point
      unsigned idx = (unsigned)(mine & 0xffffffffull);
      if (idx >= (unsigned)n) idx = 0;
      uint32_t u = (uint32_t)(mine >> 32);
      u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
      const float d = __uint_as_float(u);
      float gx, gy;
      fr.world(idx, gx, gy);
      const size_t o = ((size_t)b * T1 + t) * M + lane;
      float lx = 0.f, ly = 0.f;
#pragma unroll
      for (int e = 0; e < kMaxEdges; ++e) {  // lam = ((-R) G^T) mu   (dune.py:89); constant indices keep geo in the constant bank
        if (e < E) {
          const float m_e = smu[idx * E + e];
          lx = fmaf(fmaf(fr.sn, prm.geo.G[e][1], -fr.cs * prm.geo.G[e][0]), m_e, lx);
          ly = fmaf(fmaf(-fr.cs, prm.geo.G[e][1], -fr.sn * prm.geo.G[e][0]), m_e, ly);
          prm.sel_mu[o * E + e] = m_e;
        }
      }
      prm.sel_lam[o * 2 + 0] = lx; prm.sel_lam[o * 2 + 1] = ly;
      prm.sel_pts[o * 2 + 0] = gx; prm.sel_pts[o * 2 + 1] = gy;
      prm.sel_dist[o] = d;
      if (t == 0 && lane == 0 && prm.min_dist) prm.min_dist[b] = d;  // dune.py:97-98
    }
  }
}

// Selection for n <= 512 with the thread's own (<= 4) distance keys in registers (thread tid owns points tid + 128 j):
// per-warp REDUX rounds produce each warp's cnt smallest in ascending order, then every candidate computes its rank among
// the 4 x cnt candidates (all four warps in parallel, no serial merge) and the lanes of rank < cnt write the output rows.
__device__ __forceinline__ void select_and_write_reg(const DuneParams& prm, const ItemFrame& fr, int b, int t, int n, int cnt, int tid, uint32_t k0,
                                                     uint32_t k1, uint32_t k2, uint32_t k3, const float* smu, unsigned long long* cands) {
  const int M = prm.M, E = prm.geo.E, T1 = prm.T + 1, warp = tid >> 5, lane = tid & 31;
  unsigned long long* cand = cands + warp * M;
  for (int m = 0; m < cnt; ++m) {
    const uint32_t bd = min(min(k0, k1), min(k2, k3));
    const uint32_t md = __reduce_min_sync(0xffffffffu, bd);
    const int j = k0 == md ? 0 : (k1 == md ? 1 : (k2 == md ? 2 : 3));
    const uint32_t bi = bd == md ? (uint32_t)(tid + 128 * j) : 0xFFFFFFFFu;
    const uint32_t mi = __reduce_min_sync(0xffffffffu, bi);
    if (md != 0xFFFFFFFFu && bi == mi) {  // the owner retires the key
      if (j == 0) k0 = 0xFFFFFFFFu;
      else if (j == 1) k1 = 0xFFFFFFFFu;
      else if (j == 2) k2 = 0xFFFFFFFFu;
      else k3 = 0xFFFFFFFFu;
    }
    if (lane == 0) cand[m] = md == 0xFFFFFFFFu ? ~0ull : (((unsigned long long)md << 32) | mi);
  }
  __syncthreads();
  if (lane < cnt) {
    const unsigned long long mine = cand[lane];
    int rank = lane;  // candidates of the own warp are sorted and distinct
    for (int w = 0; w < 4; ++w) {
      if (w == warp) continue;
      for (int r = 0; r < cnt; ++r) rank += cands[w * M + r] < mine ? 1 : 0;  // keys carry the point index: no ties
    }
    if (mine != ~0ull && rank < cnt) {
      const unsigned idx = (unsigned)(mine & 0xffffffffull);
      uint32_t u = (uint32_t)(mine >> 32);
      u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
      const float d = __uint_as_float(u);
      float gx, gy;
      fr.world(idx, gx, gy);
      const size_t o = ((size_t)b * T1 + t) * M + rank;
      float lx = 0.f, ly = 0.f;
#pragma unroll
      for (int e = 0; e < kMaxEdges; ++e) {  // lam = ((-R) G^T) mu   (dune.py:89)
        if (e < E) {
          const float m_e = smu[idx * E + e];
          lx = fmaf(fmaf(fr.sn, prm.geo.G[e][1], -fr.cs * prm.geo.G[e][0]), m_e, lx);
          ly = fmaf(fmaf(-fr.cs, prm.geo.G[e][1], -fr.sn * prm.geo.G[e][0]), m_e, ly);
          prm.sel_mu[o * E + e] = m_e;
        }
      }
      prm.sel_lam[o * 2 + 0] = lx; prm.sel_lam[o * 2 + 1] = ly;
      prm.sel_pts[o * 2 + 0] = gx; prm.sel_pts[o * 2 + 1] = gy;
      prm.sel_dist[o] = d;
      if (t == 0 && rank == 0 && prm.min_dist) prm.min_dist[b] = d;  // dune.py:97-98
    }
  }
}

}  // namespace tc

// ------------------------------------------------------------------------------------------------------
// Exact kernel: two 128-point tiles ("slots") per CTA, interleaved by the same 128 threads; thread r owns point r of both
// tiles.  Per stage and slot: read the slot's D row -> LayerNorm/tanh or ReLU -> fp16 split -> A row -> barrier -> the
// warpgroup's MMAs for the slot.
template <bool kFast>
__global__ void __launch_bounds__(128) dune_tcp_kernel(const DuneParams prm, const unsigned char* __restrict__ image) {
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  using I = TcImage;
  unsigned char* simg = smem_dyn;
  unsigned char* tiles = simg + I::kBytes;
  const float* fl = reinterpret_cast<const float*>(simg + I::kFloatOff);
  unsigned char* tail = tiles + 2 * tc::kTileBytes;
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(tail);
  float* smu = reinterpret_cast<float*>(tail + (size_t)prm.N * 8);
  unsigned long long* cands = reinterpret_cast<unsigned long long*>(tail + (size_t)prm.N * 8 + (((size_t)prm.N * prm.geo.E * 4 + 7) / 8) * 8);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int prow = tc::tile_row(tid);
  for (int i = tid; i < I::kBytes / 16; i += 128) reinterpret_cast<uint4*>(simg)[i] = reinterpret_cast<const uint4*>(image)[i];
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // operand image -> visible to the tensor core (async proxy)
  __syncthreads();
  const uint32_t simg_u = tc::smem_u32(simg);

  // activations (already split) of `slot` -> the slot's tile, then the warpgroup runs the layer's MMAs on it
  auto publish = [&](const uint32_t (&hi)[16], const uint32_t (&lo)[16], int slot, int layer) {
    unsigned char* tile = tiles + slot * tc::kTileBytes;
    tc::st_a(tile, prow, hi, lo);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    tc::layer_mma<true>(tile, simg_u, layer, warp, lane);
  };

  const int T1 = prm.T + 1, N = prm.N, M = prm.M, E = prm.geo.E;
  const int items = prm.B * T1;
  const int n_work = prm.only_flagged ? *prm.flag_count : items;  // screening mode: only the items the screen could not narrow down
  for (int wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
    const int item = prm.only_flagged ? prm.flag_list[wi] : wi;
    const int b = item / T1, t = item - b * T1;
    if (prm.active && prm.active[b] == 0) continue;  // uniform per CTA
    int n = prm.num_points ? prm.num_points[b] : N;
    n = n < 0 ? 0 : (n > N ? N : n);
    const int cnt = n < M ? n : M;
    if (t == 0 && tid == 0) {
      prm.sel_count[b] = cnt;
      if (n == 0 && prm.min_dist) prm.min_dist[b] = __int_as_float(0x7f800000);
    }
    if (n == 0) continue;
    const tc::ItemFrame fr = tc::item_frame(prm, b, t);
    const bool reg_keys = n <= 512;  // the thread's own keys stay in registers (uniform per CTA)
    uint32_t k0 = 0xFFFFFFFFu, k1 = 0xFFFFFFFFu, k2 = 0xFFFFFFFFu, k3 = 0xFFFFFFFFu;

    // ---- phase 1: the network, 256 points (two slots) per pass ---------------------------------------------------------
#pragma unroll 1
    for (int base = 0; base < n; base += 256) {
      const int nslots = base + 128 < n ? 2 : 1;  // a pass whose second tile would be empty runs one slot
#pragma unroll 1
      for (int sl = 0; sl < nslots; ++sl) {  // stage 0: layer 0 (2 -> 32) on the FMA pipe + LayerNorm/tanh
        int i = base + sl * 128 + tid;
        i = i < n ? i : n - 1;
        float x0, y0;
        fr.local(i, x0, y0);
        tc::f2 hp[16];
        tc::layer0(fl, x0, y0, 0, hp);
        uint32_t hi[16], lo[16];
        tc::ln_tanh_split<kFast>(hp, fl + I::G1, fl + I::BE1, hi, lo);
        publish(hi, lo, sl, 0);
      }
#pragma unroll 1
      for (int st = 1; st < 5; ++st) {  // stage st: epilogue of dense layer st-1, operands of dense layer st (4 = head)
#pragma unroll 1
        for (int sl = 0; sl < nslots; ++sl) {
          tc::f2 hp[16];
          uint32_t hi[16], lo[16];
          tc::ld32p(tiles + sl * tc::kTileBytes, prow, hp);
          if (st & 1) tc::relu_split(hp, hi, lo);
          else tc::ln_tanh_split<kFast>(hp, fl + I::G1 + 32 * st, fl + I::BE1 + 32 * st, hi, lo);  // st = 2: G6/BE6, st = 4: G11/BE11
          publish(hi, lo, sl, st);
        }
      }
#pragma unroll 1
      for (int sl = 0; sl < nslots; ++sl) {  // head epilogue
        float mu[8];
        tc::ld8(tiles + sl * tc::kTileBytes, prow, mu);
        int i = base + sl * 128 + tid;
        const bool valid = i < n;
        i = valid ? i : n - 1;
        float x0, y0;
        fr.local(i, x0, y0);
        const uint32_t key = tc::finish_point(prm, mu, x0, y0, i, valid, E, smu, reg_keys ? nullptr : keys);
        const int j = (base >> 7) + sl;
        if (j == 0) k0 = key;
        else if (j == 1) k1 = key;
        else if (j == 2) k2 = key;
        else if (j == 3) k3 = key;
      }
    }
    __syncthreads();
    // ---- phases 2 / 3: top-M and the output rows -----------------------------------------------------------------------
    if (reg_keys) tc::select_and_write_reg(prm, fr, b, t, n, cnt, tid, k0, k1, k2, k3, smu, cands);
    else tc::select_and_write(prm, fr, b, t, n, cnt, warp, lane, keys, smu, cands);
    __syncthreads();  // smu / cands (and keys) are reused by the next item
  }
}

}  // namespace nb
