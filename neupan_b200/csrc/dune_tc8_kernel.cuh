// DUNE kernel with TWO THREADS PER POINT (8 warps per 128-point tile).
//
// Every point is shared by two threads that own 16 of the 32 features each: half the per-thread state of dune_tcp_kernel,
// twice the warps per tile, the same two 16 KB tiles per CTA.
//
//   thread (row r = tid & 127, half hf = tid >> 7): warps w and w + 4 own the same tile rows and split the columns: D features
//   [16 hf, 16 hf + 16), A K range [16 hf, 16 hf + 16).  The first warpgroup issues the layer's MMAs; a block barrier hands D to
//   both halves.  LayerNorm needs the sum of squares over all 32 features: both threads read the other half as well and add
//   the two half sums -- the same two numbers, so both get the same bits (a + b = b + a) without any exchange.  Layer 0
//   (2 -> 32, FMA pipe) is evaluated in full by both threads.  The head epilogue (mu, distance, sort key) of slot s is done by
//   the threads with hf == s.
// Everything else -- operand image, bias product, centred LayerNorm, folded tanh map, shared-reciprocal tanh, rank-merge
// top-M -- is the contract of dune_tcp_kernel.
#pragma once
#include "dune_tc_kernel.cuh"

namespace nb {
namespace tc {

// the thread's half of the A row (K 16 hf .. 16 hf + 15): chunks 2 hf, 2 hf + 1 of hi and of lo
__device__ __forceinline__ void st_a_half(unsigned char* tile, int p, int hf, const uint32_t (&hi)[8], const uint32_t (&lo)[8]) {
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    *reinterpret_cast<uint4*>(tile + chunk_off(p, 2 * hf + q)) = make_uint4(hi[4 * q], hi[4 * q + 1], hi[4 * q + 2], hi[4 * q + 3]);
    *reinterpret_cast<uint4*>(tile + chunk_off(p, 4 + 2 * hf + q)) = make_uint4(lo[4 * q], lo[4 * q + 1], lo[4 * q + 2], lo[4 * q + 3]);
  }
}

// features 16 half .. 16 half + 15 of the row's D as 8 pairs
__device__ __forceinline__ void ld16p(const unsigned char* tile, int p, int half, f2 (&hp)[8]) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const uint4 v = *reinterpret_cast<const uint4*>(tile + chunk_off(p, 4 * half + c));
    hp[2 * c] = pku(v.x, v.y);
    hp[2 * c + 1] = pku(v.z, v.w);
  }
}

// sum of squares of 16 features held as 8 packed pairs; fixed association (two chains, then lanes) so that the two threads of a
// point obtain bit-identical half sums
__device__ __forceinline__ float sumsq16(const f2 (&hp)[8]) {
  f2 qa = 0ull, qb = 0ull;
#pragma unroll
  for (int c = 0; c < 8; c += 2) {
    qa = fma2(hp[c], hp[c], qa);
    qb = fma2(hp[c + 1], hp[c + 1], qb);
  }
  float q0, q1;
  upk(add2(qa, qb), q0, q1);
  return q0 + q1;
}

// own 16 features: a = h r g + be (g, be pre-scaled by 2 log2 e), rr = 1 / (exp2(a) + 1), fp16 split (see ln_tanh_split)
template <bool kFast>
__device__ __forceinline__ void tanh_split16(const f2 (&hp)[8], float r, const float* __restrict__ g, const float* __restrict__ be, uint32_t (&hi)[8],
                                             uint32_t (&lo)[8]) {
  const f2 r2 = pk(r, r), one2 = pk(1.0f, 1.0f);
#pragma unroll
  for (int c = 0; c < 8; c += 2) {
    const ulonglong2 gg = *reinterpret_cast<const ulonglong2*>(g + 2 * c);
    const ulonglong2 bb = *reinterpret_cast<const ulonglong2*>(be + 2 * c);
    float a0, a1, a2, a3, e0, e1, e2, e3;
    upk(fma2(mul2(hp[c], r2), gg.x, bb.x), a0, a1);
    upk(fma2(mul2(hp[c + 1], r2), gg.y, bb.y), a2, a3);
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(a0));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(a1));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e2) : "f"(a2));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e3) : "f"(a3));
    const f2 da = add2(pk(e0, e1), one2), db = add2(pk(e2, e3), one2);
    float r0, r1, r2s, r3;
    if (kFast) {
      float p0, p1, t;
      upk(mul2(da, db), p0, p1);
      const float pp = p0 * p1;
      asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(pp));
      const f2 u = pk(t * p1, t * p0);
      upk(mul2(u, db), r0, r1);
      upk(mul2(u, da), r2s, r3);
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

__device__ __forceinline__ void relu_split16(const f2 (&hp)[8], uint32_t (&hi)[8], uint32_t (&lo)[8]) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    float a0, a1;
    upk(hp[c], a0, a1);
    asm("cvt.rz.relu.f16x2.f32 %0, %1, %2;" : "=r"(hi[c]) : "f"(a1), "f"(a0));
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hi[c]));
    asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(lo[c]) : "f"(__fsub_rn(a1, f.y)), "f"(__fsub_rn(a0, f.x)));
  }
}

// Selection for n <= 512 in the 8-warp kernel: thread (row, hf) keeps the keys of its points row + 128 (2 j + hf), j = 0, 1.
// Per-warp REDUX rounds give each of the 8 warps its cnt smallest in ascending order; every candidate then computes its rank
// among the 8 x cnt candidates and the lanes of rank < cnt write the output rows.
__device__ __forceinline__ void select_and_write_reg8(const DuneParams& prm, const ItemFrame& fr, int b, int t, int n, int cnt, int tid, uint32_t k0,
                                                      uint32_t k1, const float* smu, unsigned long long* cands) {
  const int M = prm.M, E = prm.geo.E, T1 = prm.T + 1, warp = tid >> 5, lane = tid & 31;
  const int row = tid & 127, hf = tid >> 7;
  unsigned long long* cand = cands + warp * M;
  for (int m = 0; m < cnt; ++m) {
    const uint32_t bd = min(k0, k1);
    const uint32_t md = __reduce_min_sync(0xffffffffu, bd);
    const int j = k0 == md ? 0 : 1;
    const uint32_t bi = bd == md ? (uint32_t)(row + 128 * (2 * j + hf)) : 0xFFFFFFFFu;
    const uint32_t mi = __reduce_min_sync(0xffffffffu, bi);
    if (md != 0xFFFFFFFFu && bi == mi) {  // the owner retires the key
      if (j == 0) k0 = 0xFFFFFFFFu;
      else k1 = 0xFFFFFFFFu;
    }
    if (lane == 0) cand[m] = md == 0xFFFFFFFFu ? ~0ull : (((unsigned long long)md << 32) | mi);
  }
  __syncthreads();
  if (lane < cnt) {
    const unsigned long long mine = cand[lane];
    int rank = lane;  // candidates of the own warp are sorted and distinct
    for (int w = 0; w < 8; ++w) {
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

// generic selection (any n): keys in shared memory, 8 warps; same algorithm as select_and_write with a stride of 256
__device__ __forceinline__ void select_and_write8(const DuneParams& prm, const ItemFrame& fr, int b, int t, int n, int cnt, int warp, int lane,
                                                  unsigned long long* keys, const float* smu, unsigned long long* cands) {
  const int M = prm.M, E = prm.geo.E, T1 = prm.T + 1;
  unsigned long long mine = ~0ull;
  {
    unsigned long long* cand = cands + warp * M;
    for (int m = 0; m < cnt; ++m) {
      unsigned bd = 0xFFFFFFFFu, bi = 0xFFFFFFFFu;
      for (int i = warp * 32 + lane; i < n; i += 256) {
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
  if (warp == 0) {  // merge the 8 candidate lists
    const int total = 8 * cnt;
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
    if (lane < cnt) {
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
      for (int e = 0; e < kMaxEdges; ++e) {
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
      if (t == 0 && lane == 0 && prm.min_dist) prm.min_dist[b] = d;
    }
  }
}

}  // namespace tc

// shared memory: operand image | two tiles | keys (N x 8 B, generic path) | smu (N x E floats) | candidates (8 warps x M)
__host__ __device__ inline size_t dune_tc8_smem_bytes(int N, int E, int M) {
  return TcImage::kBytes + 2 * (size_t)tc::kTileBytes + (size_t)N * 8 + (((size_t)N * E * 4 + 7) / 8) * 8 + (size_t)8 * M * 8 + 64;
}

template <bool kFast, int kMinBlocks>
__global__ void __launch_bounds__(256, kMinBlocks) dune_tc8_kernel(const DuneParams prm, const unsigned char* __restrict__ image) {
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
  const int row = tid & 127, hf = tid >> 7;  // hf is warp-uniform
  const int prow = tc::tile_row(row);
  for (int i = tid; i < I::kBytes / 16; i += 256) reinterpret_cast<uint4*>(simg)[i] = reinterpret_cast<const uint4*>(image)[i];
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const uint32_t simg_u = tc::smem_u32(simg);

  // both halves store their operands; the first warpgroup runs the MMAs; the block barrier after them hands D to both halves.
  // The barrier before the stores: a row's operands overwrite that row's D, which BOTH of its threads read (each needs the other
  // half's features for the LayerNorm), so neither may store until its partner has finished reading.
  auto publish = [&](const uint32_t (&hi)[8], const uint32_t (&lo)[8], int slot, int layer) {
    unsigned char* tile = tiles + slot * tc::kTileBytes;
    __syncthreads();
    tc::st_a_half(tile, prow, hf, hi, lo);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (hf == 0) tc::layer_mma<true>(tile, simg_u, layer, warp, lane);
    __syncthreads();
  };

  const int T1 = prm.T + 1, N = prm.N, M = prm.M, E = prm.geo.E;
  const int items = prm.B * T1;
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
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
    const bool reg_keys = n <= 512;
    uint32_t k0 = 0xFFFFFFFFu, k1 = 0xFFFFFFFFu;

#pragma unroll 1
    for (int base = 0; base < n; base += 256) {
      const int nslots = base + 128 < n ? 2 : 1;
#pragma unroll 1
      for (int sl = 0; sl < nslots; ++sl) {  // stage 0: layer 0 (2 -> 32, both threads in full) + LayerNorm/tanh of the own half
        int i = base + sl * 128 + row;
        i = i < n ? i : n - 1;
        float x0, y0;
        fr.local(i, x0, y0);
        tc::f2 own[8];
        float qo, qw;
        {
          tc::f2 oth[8];
          tc::layer0(fl, x0, y0, 16 * (1 - hf), oth);
          qo = tc::sumsq16(oth);
          tc::layer0(fl, x0, y0, 16 * hf, own);
          qw = tc::sumsq16(own);
        }
        float r;
        asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(fmaf(qw + qo, 1.0f / 32, 1e-5f)));
        uint32_t hi[8], lo[8];
        tc::tanh_split16<kFast>(own, r, fl + I::G1 + 16 * hf, fl + I::BE1 + 16 * hf, hi, lo);
        publish(hi, lo, sl, 0);
      }
#pragma unroll 1
      for (int st = 1; st < 5; ++st) {
#pragma unroll 1
        for (int sl = 0; sl < nslots; ++sl) {
          tc::f2 own[8];
          uint32_t hi[8], lo[8];
          const unsigned char* tile = tiles + sl * tc::kTileBytes;
          if (st & 1) {
            tc::ld16p(tile, prow, hf, own);
            tc::relu_split16(own, hi, lo);
          } else {
            float qo;
            {
              tc::f2 oth[8];
              tc::ld16p(tile, prow, 1 - hf, oth);
              qo = tc::sumsq16(oth);
            }
            tc::ld16p(tile, prow, hf, own);
            const float qw = tc::sumsq16(own);
            float r;
            asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(fmaf(qw + qo, 1.0f / 32, 1e-5f)));
            tc::tanh_split16<kFast>(own, r, fl + I::G1 + 32 * st + 16 * hf, fl + I::BE1 + 32 * st + 16 * hf, hi, lo);
          }
          publish(hi, lo, sl, st);
        }
      }
      // head epilogue: slot s by the threads with hf == s
      if (hf < nslots) {
        float mu[8];
        tc::ld8(tiles + hf * tc::kTileBytes, prow, mu);
        int i = base + hf * 128 + row;
        const bool valid = i < n;
        i = valid ? i : n - 1;
        float x0, y0;
        fr.local(i, x0, y0);
        const uint32_t key = tc::finish_point(prm, mu, x0, y0, i, valid, E, smu, reg_keys ? nullptr : keys);
        if (base == 0) k0 = key;
        else if (base == 256) k1 = key;
      }
      __syncthreads();  // D of both slots has been read before the next pass (or item) overwrites the tiles
    }
    // ---- top-M and the output rows -----------------------------------------------------------------------------------
    if (reg_keys) tc::select_and_write_reg8(prm, fr, b, t, n, cnt, tid, k0, k1, smu, cands);
    else tc::select_and_write8(prm, fr, b, t, n, cnt, warp, lane, keys, smu, cands);
    __syncthreads();  // smu / cands (and keys) are reused by the next item
  }
}

}  // namespace nb
