// DUNE with screening (NB_OPT_DUNE_KERNEL = 4): a cheap interval pass over all points, the exact network only for the few
// points that can be among the M closest.
//
// Only the M (= 10) smallest of the N (= 500) distances of an (environment, step) item are ever consumed (dune.py:100-104,
// nrmp.py:243-259), but dune_tcp_kernel pays the full fp32-accurate network -- fp16 hi/lo split, 3 MMA passes, exp2 + rcp tanh --
// for every point.  Here:
//
//  1. screening pass       (dune_screen_mma_kernel.cuh for clouds of <= 1024 points -- the default --, dune_screen_kernel below
//     otherwise or with NB_OPT_DUNE_SCREEN_MMA = 0): every point through a SINGLE-pass fp16 network (activations and weights rounded
//     to fp16 once, fp32 accumulation, tanh by MUFU.TANH: a third of the MMAs and fewer MUFU operations per point), giving an
//     approximate distance d~ and a per-point error radius eps = c_mu sum_e |G_e p0 - h_e| + 1e-4 (d is linear in mu, |mu~ - mu|
//     <= c_mu).  With tau = the M-th smallest upper bound d~ + eps, a point whose lower bound d~ - eps exceeds tau cannot be among
//     the M smallest EXACT distances; the others (typically 11-16 of 500) are the item's candidates.
//  2. dune_refine_kernel   the candidates through exactly the arithmetic of dune_tcp_kernel (same helpers, same wgmma sequence;
//     rows of an MMA tile are independent, so a point's mu / distance are bit-identical to what the full kernel computes for it);
//     work lists by candidate count (filled by the screening kernels): an item with 17..32 candidates takes a warp, two items with
//     <= 16 share one; 8 units per two-slot pass; rank-based selection inside the group, output rows.
//  3. items with more than 32 candidates (or N <= 32: no screening needed) go to the exact path: dune_tcp_kernel with
//     `only_flagged`.
// Result: the same selection, mu, lam, distances as variant 2, bit for bit (tests compare the two on every config and on the full
// C4 batch), provided c_mu bounds the screening error of the points NOT refined.  That is not left to a constant: the refine
// kernel knows the exact distance of every candidate, and an item in which any candidate's screened distance is off by more than
// half its radius is handed to the exact kernel as well; the handle's c_mu is max(0.008, 4 x a calibration measurement on this
// checkpoint) (largest error seen on the shipped checkpoints: 3.1e-3), the statistics of every launch are readable
// (`nb_pan_read_screen_stats`) and tests/test_gpu_screen.py asserts the margin.
#pragma once
#include "dune_tc_kernel.cuh"

namespace nb {

namespace tc {

// the thread's activations (single fp16 pass) -> the hi half of its A row
__device__ __forceinline__ void st_a_hi(unsigned char* tile, int p, const uint32_t (&hi)[16]) {
#pragma unroll
  for (int q = 0; q < 4; ++q)
    *reinterpret_cast<uint4*>(tile + chunk_off(p, q)) = make_uint4(hi[4 * q], hi[4 * q + 1], hi[4 * q + 2], hi[4 * q + 3]);
}

// LayerNorm (centred inputs, eps 1e-5) + tanh by MUFU.TANH; g / be are the checkpoint's plain gain / offset
__device__ __forceinline__ void ln_tanh_screen(const f2 (&hp)[16], const float* __restrict__ g, const float* __restrict__ be, uint32_t (&hi)[16]) {
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
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(fmaf(q0 + q1, 1.0f / 32, 1e-5f)));
  const f2 r2 = pk(r, r);
#pragma unroll
  for (int c = 0; c < 16; c += 2) {
    const ulonglong2 gg = *reinterpret_cast<const ulonglong2*>(g + 2 * c);
    const ulonglong2 bb = *reinterpret_cast<const ulonglong2*>(be + 2 * c);
    float a0, a1, a2, a3;
    upk(fma2(mul2(hp[c], r2), gg.x, bb.x), a0, a1);
    upk(fma2(mul2(hp[c + 1], r2), gg.y, bb.y), a2, a3);
    // MUFU.TANH on f32 (one MUFU per feature either way: the f16x2 form is two MUFUs plus byte permutes), then one pack per pair
    float t0, t1, t2, t3;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t0) : "f"(a0));
    asm("tanh.approx.f32 %0, %1;" : "=f"(t1) : "f"(a1));
    asm("tanh.approx.f32 %0, %1;" : "=f"(t2) : "f"(a2));
    asm("tanh.approx.f32 %0, %1;" : "=f"(t3) : "f"(a3));
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(hi[c]) : "f"(t1), "f"(t0));
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(hi[c + 1]) : "f"(t3), "f"(t2));
  }
}

__device__ __forceinline__ void relu_screen(const f2 (&hp)[16], uint32_t (&hi)[16]) {
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    float a0, a1;
    upk(hp[c], a0, a1);
    asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(hi[c]) : "f"(a1), "f"(a0));
  }
}

// smallest value above k whose low 9 bits carry the point's index in the item (< 512): keys become unique, so a REDUX round
// removes exactly one entry and needs no second reduction over indices.  Rounding a bound UP only widens the candidate set.
__device__ __forceinline__ uint32_t unique_key(uint32_t k, int idx) { return ((min(k, 0xFFFFF000u) + 0x200u) & ~0x1FFu) | (uint32_t)idx; }

// d~ = relu(mu)^T (G p0 - h) and sum_e |G_e p0 - h_e| (the factor of the error radius)
template <int kE>
__device__ __forceinline__ void screen_distance(const DuneParams& prm, const float (&mu)[8], float2 xy, int E, float& d, float& sa) {
#pragma unroll
  for (int e = 0; e < kE; ++e) {
    if (e < E) {
      const float ge = fmaf(prm.geo.G[e][1], xy.y, prm.geo.G[e][0] * xy.x) - prm.geo.h[e];
      d = fmaf(fmaxf(mu[e], 0.f), ge, d);
      sa += fabsf(ge);
    }
  }
}

// one thread: item -> the refine list of its size class (dune_refine_kernel packs two items of <= 16 candidates into one warp)
__device__ __forceinline__ void refine_append(const DuneParams& prm, int item, int nc) {
  if (nc <= 0) return;
  const int big = nc > 16 ? 1 : 0;
  const int pos = atomicAdd(prm.flag_count + 1 + big, 1);
  prm.refine_list[(size_t)big * prm.B * (prm.T + 1) + pos] = item;
}

__device__ __forceinline__ void cp_async4(const float* smem_dst, const float* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

}  // namespace tc

// shared memory of the screen kernel: operand image | two tiles | UB keys (N x 8) | lower bounds (N x 4) | d~ (N x 4) |
// per-warp candidates (4 M x 8)
__host__ __device__ inline size_t dune_screen_smem_bytes(int N, int M) {
  return TcImage::kBytes + 2 * (size_t)tc::kTileBytes + (size_t)N * 16 + (size_t)4 * M * 8 + 64;
}

template <int kDummy>
__global__ void __launch_bounds__(128) dune_screen_kernel(const DuneParams prm, const unsigned char* __restrict__ image) {
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  using I = TcImage;
  unsigned char* simg = smem_dyn;
  unsigned char* tiles = simg + I::kBytes;
  const float* fl = reinterpret_cast<const float*>(simg + I::kFloatOff);
  unsigned char* tail = tiles + 2 * tc::kTileBytes;
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(tail);  // (orderable(UB) << 32) | index
  float* lbv = reinterpret_cast<float*>(tail + (size_t)prm.N * 8);
  float* dtv = lbv + prm.N;
  unsigned long long* cands = reinterpret_cast<unsigned long long*>(tail + (size_t)prm.N * 16);
  __shared__ uint32_t tau_s;
  __shared__ int cnt_s;
  __shared__ int list_s[kCandMax];
  __shared__ float ldt_s[kCandMax], lrad_s[kCandMax];
  __shared__ float2 xy_s[2][128];  // robot-frame coordinates of the points in flight (stage 0 -> head)

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int prow = tc::tile_row(tid);
  for (int i = tid; i < I::kBytes / 16; i += 128) reinterpret_cast<uint4*>(simg)[i] = reinterpret_cast<const uint4*>(image)[i];
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const uint32_t simg_u = tc::smem_u32(simg);

  auto publish = [&](const uint32_t (&hi)[16], int slot, int layer) {
    unsigned char* tile = tiles + slot * tc::kTileBytes;
    tc::st_a_hi(tile, prow, hi);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    tc::layer_mma<false>(tile, simg_u, layer, warp, lane);
  };

  const int T1 = prm.T + 1, N = prm.N, M = prm.M, E = prm.geo.E;
  const int items = prm.B * T1;
  // Items with n <= 512 keep their bounds in registers; the key arrays then stage the raw point data (x | y | vx | vy, N floats
  // each), copied asynchronously (cp.async, each thread exactly the <= 4 entries it reads itself: no barrier) -- for the NEXT
  // item as soon as the last stage 0 of the current one has consumed the buffer, so the point loads never sit on the critical path.
  float* raw = reinterpret_cast<float*>(keys);
  int staged = -1;  // item whose points are in (or on their way into) `raw`
  auto stage_points = [&](int it) -> bool {
    const int bb = it / T1;
    int nn = prm.num_points ? prm.num_points[bb] : N;
    nn = nn > N ? N : nn;
    if ((nn <= kCandMax && !prm.calibrate) || nn > 512 || nn <= 0) return false;
    const float* px = prm.points + (size_t)bb * 2 * N;
    const float* vx = prm.velocities ? prm.velocities + (size_t)bb * 2 * N : nullptr;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = tid + 128 * j;
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
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int b = item / T1, t = item - b * T1;
    if (prm.skip_t0 && t == 0) {  // same inputs as in the previous PAN iteration: its outputs stand
      if (tid == 0) prm.cand_cnt[item] = 0;
      continue;
    }
    int32_t* out_idx = prm.cand_idx + (size_t)item * kCandMax;
    float* out_dt = prm.cand_dt + (size_t)item * kCandMax;
    // the item's header values are loaded together (one memory latency, not three dependent ones)
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
    const bool reg_keys = n <= 512;  // the thread's (<= 4) bounds stay in registers; larger items use the shared-memory arrays
    if (reg_keys) {
      if (staged != item) {
        tc::cp_async_wait_all();  // an abandoned copy (its item was skipped) must not land after this one
        stage_points(item);
        staged = item;
      }
      tc::cp_async_wait_all();
    }
    uint32_t k0 = 0xFFFFFFFFu, k1 = 0xFFFFFFFFu, k2 = 0xFFFFFFFFu, k3 = 0xFFFFFFFFu;
    float l0 = 0.f, l1 = 0.f, l2 = 0.f, l3 = 0.f, d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;

#pragma unroll 1
    for (int base = 0; base < n; base += 256) {
      const int nslots = base + 128 < n ? 2 : 1;
#pragma unroll 1
      for (int sl = 0; sl < nslots; ++sl) {
        int i = base + sl * 128 + tid;
        float x0 = 0.f, y0 = 0.f;
        if (!reg_keys) {
          fr.local(i < n ? i : n - 1, x0, y0);
        } else if (i < n) {  // rows beyond n run on zeros (their results are never looked at)
          float gx = raw[i], gy = raw[N + i];
          if (fr.vx) {
            gx = flow(gx, raw[2 * N + i], fr.dt, fr.t);
            gy = flow(gy, raw[3 * N + i], fr.dt, fr.t);
          }
          const float dx = gx - fr.sx, dy = gy - fr.sy;
          x0 = fmaf(fr.cs, dx, fr.sn * dy);
          y0 = fmaf(fr.cs, dy, -(fr.sn * dx));
        }
        xy_s[sl][tid] = make_float2(x0, y0);
        tc::f2 hp[16];
        tc::layer0(fl, x0, y0, 0, hp);
        uint32_t hi[16];
        tc::ln_tanh_screen(hp, fl + I::G1, fl + I::BE1, hi);
        publish(hi, sl, 0);
      }
      if (reg_keys && base + 256 >= n && item + (int)gridDim.x < items) {  // `raw` is free: start on the next item's points
        if (stage_points(item + (int)gridDim.x)) staged = item + (int)gridDim.x;
      }
#pragma unroll 1
      for (int st = 1; st < 5; ++st) {
#pragma unroll 1
        for (int sl = 0; sl < nslots; ++sl) {
          tc::f2 hp[16];
          uint32_t hi[16];
          tc::ld32p(tiles + sl * tc::kTileBytes, prow, hp);
          if (st & 1) tc::relu_screen(hp, hi);
          else tc::ln_tanh_screen(hp, fl + I::G1 + 32 * st, fl + I::BE1 + 32 * st, hi);
          publish(hi, sl, st);
        }
      }
#pragma unroll 1
      for (int sl = 0; sl < nslots; ++sl) {  // head: approximate distance and its error radius
        float mu[8];
        tc::ld8(tiles + sl * tc::kTileBytes, prow, mu);
        const int i = base + sl * 128 + tid;
        uint32_t kub = 0xFFFFFFFFu;
        float lbi = __int_as_float(0x7f800000), dti = 0.f;
        if (i < n) {
          const float2 xy = xy_s[sl][tid];
          float d = 0.f, sa = 0.f;
          if (E == 4) tc::screen_distance<4>(prm, mu, xy, 4, d, sa);  // every shipped robot: no per-edge branches
          else tc::screen_distance<kMaxEdges>(prm, mu, xy, E, d, sa);
          const float eps = fmaf(prm.c_mu, sa, 1e-4f);
          kub = orderable(d + eps); lbi = d - eps; dti = d;
          if (reg_keys) kub = tc::unique_key(kub, i);
          if (!reg_keys) {
            keys[i] = ((unsigned long long)kub << 32) | (unsigned)i;
            lbv[i] = lbi;
            dtv[i] = dti;
          }
        }
        const int j = (base >> 7) + sl;  // the thread's j-th point (n <= 512: at most four)
        if (j == 0) { k0 = kub; l0 = lbi; d0 = dti; }
        else if (j == 1) { k1 = kub; l1 = lbi; d1 = dti; }
        else if (j == 2) { k2 = kub; l2 = lbi; d2 = dti; }
        else if (j == 3) { k3 = kub; l3 = lbi; d3 = dti; }
      }
    }
    if (tid == 0) cnt_s = 0;
    __syncthreads();
    if (n <= kCandMax) {  // calibration mode: all points, with their screened distance
      if (tid < n) { out_idx[tid] = tid; out_dt[tid] = d0; }
      if (tid == 0) { prm.cand_cnt[item] = n; tc::refine_append(prm, item, n); }
      __syncthreads();
      continue;
    }
    // ---- tau = the M-th smallest upper bound
    uint32_t tau;
    if (reg_keys) {
      // unique 32-bit keys: M REDUX rounds per warp (each removes the one entry that equals the minimum), then every warp merges
      // the 4 M survivors the same way -- no index reduction, no rank loop, no broadcast of tau through shared memory
      uint32_t* c32 = reinterpret_cast<uint32_t*>(cands);
      uint32_t q0 = k0, q1 = k1, q2 = k2, q3 = k3;
      for (int m = 0; m < M; ++m) {
        const uint32_t md = __reduce_min_sync(0xffffffffu, min(min(q0, q1), min(q2, q3)));
        q0 = q0 == md ? 0xFFFFFFFFu : q0; q1 = q1 == md ? 0xFFFFFFFFu : q1;
        q2 = q2 == md ? 0xFFFFFFFFu : q2; q3 = q3 == md ? 0xFFFFFFFFu : q3;
        if (lane == 0) c32[warp * M + m] = md;
      }
      __syncthreads();
      const int nc4 = 4 * M;  // <= 128 (M <= 32)
      q0 = lane < nc4 ? c32[lane] : 0xFFFFFFFFu;
      q1 = lane + 32 < nc4 ? c32[lane + 32] : 0xFFFFFFFFu;
      q2 = lane + 64 < nc4 ? c32[lane + 64] : 0xFFFFFFFFu;
      q3 = lane + 96 < nc4 ? c32[lane + 96] : 0xFFFFFFFFu;
      uint32_t md = 0xFFFFFFFFu;
      for (int m = 0; m < M; ++m) {  // n > kCandMax >= M: M finite keys exist
        md = __reduce_min_sync(0xffffffffu, min(min(q0, q1), min(q2, q3)));
        q0 = q0 == md ? 0xFFFFFFFFu : q0; q1 = q1 == md ? 0xFFFFFFFFu : q1;
        q2 = q2 == md ? 0xFFFFFFFFu : q2; q3 = q3 == md ? 0xFFFFFFFFu : q3;
      }
      tau = md;
    } else {
      // per-warp REDUX rounds over the keys in shared memory (destroying them), then rank among the 4 M candidates
      unsigned long long* cand = cands + warp * M;
      for (int m = 0; m < M; ++m) {
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
      __syncthreads();
      if (lane < M) {
        const unsigned long long mine = cands[warp * M + lane];
        int rank = lane;
        for (int w = 0; w < 4; ++w) {
          if (w == warp) continue;
          for (int r = 0; r < M; ++r) rank += cands[w * M + r] < mine ? 1 : 0;
        }
        if (mine != ~0ull && rank == M - 1) tau_s = (uint32_t)(mine >> 32);  // n > kCandMax >= M: M finite keys exist
      }
      __syncthreads();
      tau = tau_s;
    }
    if (reg_keys) {
      auto take = [&](uint32_t k, float lb, float dt, int j) {
        if (k != 0xFFFFFFFFu && orderable(lb) <= tau) {
          const int pos = atomicAdd(&cnt_s, 1);
          if (pos < kCandMax) { list_s[pos] = tid + 128 * j; ldt_s[pos] = dt; lrad_s[pos] = dt - lb; }
        }
      };
      take(k0, l0, d0, 0); take(k1, l1, d1, 1); take(k2, l2, d2, 2); take(k3, l3, d3, 3);
    } else {
      for (int i = tid; i < n; i += 128) {
        if (orderable(lbv[i]) <= tau) {
          const int pos = atomicAdd(&cnt_s, 1);
          if (pos < kCandMax) { list_s[pos] = i; ldt_s[pos] = dtv[i]; lrad_s[pos] = dtv[i] - lbv[i]; }
        }
      }
    }
    __syncthreads();
    const int nc = cnt_s;
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
    __syncthreads();  // keys / lbv / list are reused by the next item
  }
}

// ------------------------------------------------------------------------------------------------------------------------
// Exact evaluation of the candidates.  Work units come from the two lists the screen kernels fill: an item with 17..32 candidates
// takes a warp, two items with <= 16 candidates share one (lanes 0-15 / 16-31) -- the typical item has 11-16 candidates, so the
// paired form nearly halves the number of 128-row tiles.  8 units per two-slot pass (slot s, warp w -> unit 8 g + 4 s + w), lane =
// candidate.  Rows of an MMA tile are independent, so where a candidate sits does not change its mu / distance by a bit.
template <bool kFast>
__global__ void __launch_bounds__(128) dune_refine_kernel(const DuneParams prm, const unsigned char* __restrict__ image) {
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  using I = TcImage;
  unsigned char* simg = smem_dyn;
  unsigned char* tiles = simg + I::kBytes;
  const float* fl = reinterpret_cast<const float*>(simg + I::kFloatOff);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int prow = tc::tile_row(tid);
  for (int i = tid; i < I::kBytes / 16; i += 128) reinterpret_cast<uint4*>(simg)[i] = reinterpret_cast<const uint4*>(image)[i];
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const uint32_t simg_u = tc::smem_u32(simg);

  auto publish = [&](const uint32_t (&hi)[16], const uint32_t (&lo)[16], int slot, int layer) {
    unsigned char* tile = tiles + slot * tc::kTileBytes;
    tc::st_a(tile, prow, hi, lo);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    tc::layer_mma<true>(tile, simg_u, layer, warp, lane);
  };

  const int T1 = prm.T + 1, M = prm.M, E = prm.geo.E;
  const int items = prm.B * T1;
  const int nA = prm.flag_count[1], nB = prm.flag_count[2];  // items with <= 16 / with 17..32 candidates
  const int units = nB + ((nA + 1) >> 1);
  const int groups = (units + 7) >> 3;
  const int half = lane >> 4;
  for (int g = blockIdx.x; g < groups; g += gridDim.x) {
    int myitem[2], myidx[2], myli[2];  // the lane's item (-1: none), its point, its position in the item's candidate list (-1: not a candidate)
#pragma unroll
    for (int sl = 0; sl < 2; ++sl) {
      const int u = 8 * g + 4 * sl + warp;
      int it = -1, li = lane;
      if (u < nB) it = prm.refine_list[items + u];
      else if (u < units) {
        const int q = 2 * (u - nB) + half;
        it = q < nA ? prm.refine_list[q] : -1;
        li = lane & 15;
      }
      int c = it >= 0 ? prm.cand_cnt[it] : 0;
      c = c > 0 ? c : 0;
      myitem[sl] = it;
      myli[sl] = li < c ? li : -1;
      myidx[sl] = c > 0 ? prm.cand_idx[(size_t)it * kCandMax + (li < c ? li : 0)] : 0;  // idle rows run on a valid point of the item
    }
#pragma unroll 1
    for (int sl = 0; sl < 2; ++sl) {  // stage 0
      const int it = myitem[sl] >= 0 ? myitem[sl] : 0;
      const tc::ItemFrame fr = tc::item_frame(prm, it / T1, it % T1);
      float x0, y0;
      fr.local(myidx[sl], x0, y0);
      tc::f2 hp[16];
      tc::layer0(fl, x0, y0, 0, hp);
      uint32_t hi[16], lo[16];
      tc::ln_tanh_split<kFast>(hp, fl + I::G1, fl + I::BE1, hi, lo);
      publish(hi, lo, sl, 0);
    }
#pragma unroll 1
    for (int st = 1; st < 5; ++st) {
#pragma unroll 1
      for (int sl = 0; sl < 2; ++sl) {
        tc::f2 hp[16];
        uint32_t hi[16], lo[16];
        tc::ld32p(tiles + sl * tc::kTileBytes, prow, hp);
        if (st & 1) tc::relu_split(hp, hi, lo);
        else tc::ln_tanh_split<kFast>(hp, fl + I::G1 + 32 * st, fl + I::BE1 + 32 * st, hi, lo);
        publish(hi, lo, sl, st);
      }
    }
#pragma unroll 1
    for (int sl = 0; sl < 2; ++sl) {  // head, selection inside the lane's group (warp or half warp), output rows
      float mu[8];
      tc::ld8(tiles + sl * tc::kTileBytes, prow, mu);
      const int u = 8 * g + 4 * sl + warp;
      if (u >= units) continue;  // warp-uniform
      const bool whole = u < nB;  // warp-uniform
      const bool valid = myli[sl] >= 0;
      const int it = myitem[sl] >= 0 ? myitem[sl] : 0, b = it / T1, t = it - b * T1;
      const tc::ItemFrame fr = tc::item_frame(prm, b, t);
      const int idx = myidx[sl];
      float x0, y0;
      fr.local(idx, x0, y0);
      float d = 0.f, sa = 0.f;
#pragma unroll
      for (int e = 0; e < kMaxEdges; ++e) {
        if (e < E) {
          mu[e] = fmaxf(mu[e], 0.f);
          const float ge = fmaf(prm.geo.G[e][1], y0, prm.geo.G[e][0] * x0) - prm.geo.h[e];
          d = fmaf(mu[e], ge, d);
          sa += fabsf(ge);
        }
      }
      const unsigned gmask = whole ? 0xffffffffu : (half ? 0xffff0000u : 0x0000ffffu);
      bool live = valid;
      {  // the screening error on the candidates (NaN marks unscreened items): statistics, and the run-time check of the bound --
         // a candidate whose screened distance is off by more than HALF its assumed radius sends the whole item to the exact kernel
         // (which runs after this one), so the selection never rests on an error bound that the item itself contradicts
        const float dt = prm.cand_dt[(size_t)it * kCandMax + (valid ? myli[sl] : 0)];
        const bool screened = valid && dt == dt;
        const float err = screened ? fabsf(dt - d) : 0.f;
        float ratio = screened ? err / fmaxf(sa, 1e-6f) : 0.f;
        const bool viol = screened && !prm.calibrate && err > 0.5f * prm.cand_rad[(size_t)it * kCandMax + myli[sl]];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ratio = fmaxf(ratio, __shfl_xor_sync(0xffffffffu, ratio, o));
        if (lane == 0 && ratio > 0.f) atomicMax(&prm.screen_stats[0], __float_as_uint(ratio));
        if ((__ballot_sync(0xffffffffu, viol) & gmask) != 0u) {  // uniform within the group
          if (myli[sl] == 0) {
            prm.cand_cnt[it] = -1;
            atomicAdd(&prm.screen_stats[1], 1u);
            prm.flag_list[atomicAdd(prm.flag_count, 1)] = it;
          }
          live = false;
        }
      }
      // rank of the lane's (distance, point index) among its group's candidates: ascending distance, ties -> lower point index,
      // NaN distances last and never selected (like select_and_write_reg)
      const uint32_t key = live ? orderable(d) : 0xFFFFFFFFu;
      int rank = 0;
      const int gbase = whole ? 0 : (lane & 16), gsz = whole ? 32 : 16;
#pragma unroll 4
      for (int j = 0; j < gsz; ++j) {
        const uint32_t kj = __shfl_sync(0xffffffffu, key, gbase + j);
        const int ij = __shfl_sync(0xffffffffu, idx, gbase + j);
        rank += (kj < key || (kj == key && ij < idx)) ? 1 : 0;
      }
      int n_b = prm.num_points ? prm.num_points[b] : prm.N;
      n_b = n_b < 0 ? 0 : (n_b > prm.N ? prm.N : n_b);
      const int cnt_out = n_b < M ? n_b : M;
      if (key != 0xFFFFFFFFu && rank < cnt_out) {
        float gx, gy;
        fr.world(idx, gx, gy);
        const size_t o = ((size_t)b * T1 + t) * M + rank;
        float lx = 0.f, ly = 0.f;
#pragma unroll
        for (int e = 0; e < kMaxEdges; ++e) {  // lam = ((-R) G^T) mu   (dune.py:89)
          if (e < E) {
            lx = fmaf(fmaf(fr.sn, prm.geo.G[e][1], -fr.cs * prm.geo.G[e][0]), mu[e], lx);
            ly = fmaf(fmaf(-fr.cs, prm.geo.G[e][1], -fr.sn * prm.geo.G[e][0]), mu[e], ly);
            prm.sel_mu[o * E + e] = mu[e];
          }
        }
        prm.sel_lam[o * 2 + 0] = lx; prm.sel_lam[o * 2 + 1] = ly;
        prm.sel_pts[o * 2 + 0] = gx; prm.sel_pts[o * 2 + 1] = gy;
        prm.sel_dist[o] = d;
        if (t == 0 && rank == 0 && prm.min_dist) prm.min_dist[b] = d;  // dune.py:97-98
      }
    }
    __syncthreads();  // D of both slots has been read before the next group's operands arrive
  }
}

}  // namespace nb
