// Reactive obstacles of the batched world: this project's reading of IR-SIM's `rvo` behaviour with `wander` (the obstacles of
// example/dyna_obs/*/env.yaml and example/dyna_non_obs/*/env.yaml), run before world_step_kernel in nb_world_step.  IR-SIM is not
// a dependency, so the behaviour is defined here; per reactive obstacle i (behaviour kind 1), from the states at the start of the step:
//
//   1. goal       |goal - c_i| < goal_threshold: with wander a new goal is drawn uniformly in the environment's rectangle (draw n of
//                 the obstacle's counter-based SplitMix64 stream, below); without it the obstacle parks (velocity 0, still a
//                 neighbour of the others).  The initial goal is the scene's, or draw 0.
//   2. v_des      speed * (goal - c_i) / |goal - c_i|  (0 when the goal is the centre)
//   3. neighbours every other obstacle of the environment and each of its K robots whose centre lies within neighbor_range of c_i
//                 (distance <= neighbor_range; a neighbour at the same centre is skipped), each a circle: a circle's radius, a
//                 polygon's or outline's circumradius about its centre, a robot's circumradius about its state point.  A robot's
//                 velocity is 0 once collided, else that of this step's action in the world frame (diff / acker v (cos th, sin th),
//                 omni (vx, vy)).  The robots are the rows after the obstacles, in robot order.
//   4. cones      apex (v_i + v_j) / 2 (RVO); R = r_i + r_j, D = |c_j - c_i|, D' = max(D, R); edges: the unit direction to j turned by
//                 +-alpha with sin alpha = R / D', cos alpha = sqrt(D'^2 - R^2) / D' (IR-SIM's atan2 / asin / cos / sin construction
//                 without trigonometry: equal in exact arithmetic, correctly rounded here).  w = v - apex is inside when
//                 cross(left, w) <= 0 and cross(right, w) >= 0 (IR-SIM's between_vector).
//   5. candidates per axis [max(v - acce, -vmax), min(v + acce, vmax)) in steps of grid: lo + k grid, k < ceil((hi - lo) / grid)
//                 (at most 64), vx-major (index kx ny + ky); a candidate whose norm is below min_speed is skipped.
//   6. selection  the candidate outside every cone with the smallest |v - v_des|; if there is none, the smallest
//                 factor / tc_min + |v - v_des| (tc: time to collision with a neighbour, 0 when already within R, inf without a
//                 root t > 0); ties go to the lower index; no candidate at all: the velocity is unchanged.
//   7. motion     the chosen velocity goes into the obstacle's row; world_step_kernel then moves it and applies the mirror rule.
//
// Stated differences from IR-SIM: the update is Jacobi (every velocity from the states at the start of the step; IR-SIM steps its
// objects one after another), obstacles are holonomic (IR-SIM turns its diff obstacles towards the chosen velocity), every neighbour
// is a circle, and the candidate values are lo + k grid (np.arange can differ in the last bit).
//
// FP64 with explicit rounding (dmul / dadd / dsub of world_kernel.cuh, __ddiv_rn, __dsqrt_rn), so that tests/world_rvo_oracle.py
// agrees bit for bit; the one difference is CUDA's sincos for the robot's velocity.
//
// Kernel: one CTA per environment (grid-stride).  Shared memory holds the environment's centres, velocities and radii (the K robots
// last); one warp per reactive obstacle builds its neighbours' cone list by ballot compaction, then the lanes take the candidates and
// a warp reduction on (key, index) picks the winner; a ballot decides whether the penalty pass is needed.
#pragma once
#include <climits>
#include <cstdint>

#include "world_kernel.cuh"

namespace nb {

constexpr int kWorldBehCols = 13;  // kind, vxmax, vymax, acce, factor, speed, wander, goal x, y, goal_threshold, neighbor_range,
                                   // grid, min_speed
constexpr int kWorldRvoWarps = 8;
constexpr int kWorldRvoMaxAxis = 64;  // candidates per axis
constexpr uint64_t kSplitMixGamma = 0x9E3779B97F4A7C15ull;

struct WorldRvoParams {
  const double* beh;     // (O, kWorldBehCols)
  const double* radius;  // (O) circle radius, or the polygon's circumradius about its centre
  double* goal;          // (O, 2)
  int32_t* draws;        // (O) goals drawn so far
  const float* action;   // (B K, 2) this step's action
  uint64_t seed;
  double robot_r;        // circumradius of the robot polygon about its state point
  int cap;               // shared rows per environment: the largest obstacle count + K (the robots)
};

// SplitMix64 (Steele, Lea and Flood 2014): output n of the generator seeded with s is mix(s + (n + 1) gamma), so any draw is
// computed directly from its counter.
__host__ __device__ __forceinline__ uint64_t splitmix64_mix(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint64_t splitmix64_at(uint64_t s, uint64_t n) { return splitmix64_mix(s + (n + 1) * kSplitMixGamma); }
// the stream of obstacle i (index within its environment) of environment b
__host__ __device__ __forceinline__ uint64_t world_rvo_key(uint64_t seed, int b, int i) {
  return splitmix64_mix(splitmix64_mix(seed + kSplitMixGamma) ^ (((uint64_t)(uint32_t)b << 32) | (uint64_t)(uint32_t)i));
}
// (x >> 11) 2^-53: uniform in [0, 1), exact
__host__ __device__ __forceinline__ double world_u01(uint64_t x) { return (double)(x >> 11) * 0x1.0p-53; }

__device__ __forceinline__ int world_rvo_count(double lo, double hi, double grid) {
  if (!(hi > lo)) return 0;
  const double n = ceil(__ddiv_rn(dsub(hi, lo), grid));
  return n < (double)kWorldRvoMaxAxis ? (int)n : kWorldRvoMaxAxis;
}

// time to collision of p - w t with a circle of radius R about the origin: 0 when |p| <= R, inf without a root t > 0, else the
// smaller root of |w|^2 t^2 - 2 (p.w) t + |p|^2 - R^2 = 0
__device__ __forceinline__ double world_rvo_tc(double px, double py, double wx, double wy, double R) {
  const double c = dsub(ddot(px, py, px, py), dmul(R, R));
  if (c <= 0.0) return 0.0;
  const double a = ddot(wx, wy, wx, wy), pw = ddot(px, py, wx, wy);
  if (a == 0.0) return INFINITY;
  const double disc = dsub(dmul(pw, pw), dmul(a, c));
  if (disc < 0.0) return INFINITY;
  const double t = __ddiv_rn(dsub(pw, __dsqrt_rn(disc)), a);
  return t > 0.0 ? t : INFINITY;
}

// warp argmin of (key, index): every lane ends with the smallest key, the lower index on ties
__device__ __forceinline__ void world_rvo_argmin(double& key, int& idx) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    const double k2 = __shfl_xor_sync(0xffffffffu, key, m);
    const int i2 = __shfl_xor_sync(0xffffffffu, idx, m);
    if (k2 < key || (k2 == key && i2 < idx)) { key = k2; idx = i2; }
  }
}

__global__ void __launch_bounds__(32 * kWorldRvoWarps) world_rvo_kernel(const WorldParams prm, const WorldRvoParams rp) {
  extern __shared__ double rsm[];
  const int cap = rp.cap, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double* s_cx = rsm;
  double* s_cy = s_cx + cap;
  double* s_vx = s_cy + cap;
  double* s_vy = s_vx + cap;
  double* s_r = s_vy + cap;
  double* c_ax = s_r + cap + (size_t)wid * 6 * cap;  // this warp's cone list: apex, left edge, right edge
  double* c_ay = c_ax + cap;
  double* c_lx = c_ay + cap;
  double* c_ly = c_lx + cap;
  double* c_rx = c_ly + cap;
  double* c_ry = c_rx + cap;
  int32_t* nbr = reinterpret_cast<int32_t*>(s_r + cap + (size_t)kWorldRvoWarps * 6 * cap) + (size_t)wid * cap;
  for (int b = blockIdx.x; b < prm.B; b += gridDim.x) {
    const int o0 = prm.obs_begin[b], n = prm.obs_begin[b + 1] - o0;
    __syncthreads();  // the previous environment's warps are done with the shared rows
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
      const double* row = prm.obs + (size_t)kWorldObsCols * (o0 + j);
      s_cx[j] = row[0]; s_cy[j] = row[1]; s_vx[j] = row[2]; s_vy[j] = row[3]; s_r[j] = rp.radius[o0 + j];
    }
    for (int k = threadIdx.x; k < prm.K; k += blockDim.x) {  // robot k, row n + k: its state point and the velocity of this step's
      const size_t r = (size_t)b * prm.K + k;               // action (the step kernels' sincos)
      const double th = prm.states[3 * r + 2];
      double rvx = 0.0, rvy = 0.0;
      if (prm.collided[r] == 0) {
        const double a0 = (double)rp.action[2 * r], a1 = (double)rp.action[2 * r + 1];
        if (prm.kinematics == 2) {
          rvx = a0; rvy = a1;
        } else {
          double sn, cs;
          sincos(th, &sn, &cs);
          rvx = dmul(a0, cs); rvy = dmul(a0, sn);
        }
      }
      s_cx[n + k] = prm.states[3 * r]; s_cy[n + k] = prm.states[3 * r + 1]; s_vx[n + k] = rvx; s_vy[n + k] = rvy; s_r[n + k] = rp.robot_r;
    }
    __syncthreads();
    for (int i = wid; i < n; i += kWorldRvoWarps) {
      const int o = o0 + i;
      const double* beh = rp.beh + (size_t)kWorldBehCols * o;
      if (beh[0] != 1.0) continue;  // warp-uniform
      const double* env = prm.env + (size_t)kWorldEnvCols * b;
      const double cx = s_cx[i], cy = s_cy[i], vx = s_vx[i], vy = s_vy[i], ri = s_r[i];
      double gx = rp.goal[2 * o], gy = rp.goal[2 * o + 1];
      int draws = rp.draws[o];
      double dx = dsub(gx, cx), dy = dsub(gy, cy), dist = __dsqrt_rn(ddot(dx, dy, dx, dy));
      bool parked = false;
      if (dist < beh[9]) {
        if (beh[6] != 0.0) {  // wander: draw n takes the stream's values 2n and 2n + 1
          const uint64_t key = world_rvo_key(rp.seed, b, i);
          gx = dadd(env[0], dmul(world_u01(splitmix64_at(key, 2 * (uint64_t)draws)), dsub(env[2], env[0])));
          gy = dadd(env[1], dmul(world_u01(splitmix64_at(key, 2 * (uint64_t)draws + 1)), dsub(env[3], env[1])));
          ++draws;
          dx = dsub(gx, cx); dy = dsub(gy, cy); dist = __dsqrt_rn(ddot(dx, dy, dx, dy));
        } else {
          parked = true;
        }
      }
      double nvx = 0.0, nvy = 0.0;
      if (!parked) {
        double desx = 0.0, desy = 0.0;
        if (dist > 0.0) { desx = __ddiv_rn(dmul(beh[5], dx), dist); desy = __ddiv_rn(dmul(beh[5], dy), dist); }
        // the neighbours' cones, compacted by ballot in neighbour order
        int m = 0;
        const int rows = n + prm.K;
        for (int base = 0; base < rows; base += 32) {
          const int j = base + lane;
          bool take = false;
          double px = 0.0, py = 0.0, D = 0.0;
          if (j < rows && j != i) {
            px = dsub(s_cx[j], cx); py = dsub(s_cy[j], cy);
            D = __dsqrt_rn(ddot(px, py, px, py));
            take = D > 0.0 && D <= beh[10];
          }
          const unsigned mask = __ballot_sync(0xffffffffu, take);
          if (take) {
            const int q = m + __popc(mask & ((1u << lane) - 1u));
            const double R = dadd(ri, s_r[j]), Dp = D > R ? D : R;
            const double sa = __ddiv_rn(R, Dp), ca = __ddiv_rn(__dsqrt_rn(dsub(dmul(Dp, Dp), dmul(R, R))), Dp);
            const double ux = __ddiv_rn(px, D), uy = __ddiv_rn(py, D);
            c_ax[q] = dmul(0.5, dadd(vx, s_vx[j])); c_ay[q] = dmul(0.5, dadd(vy, s_vy[j]));
            c_lx[q] = dsub(dmul(ux, ca), dmul(uy, sa)); c_ly[q] = dadd(dmul(ux, sa), dmul(uy, ca));
            c_rx[q] = dadd(dmul(ux, ca), dmul(uy, sa)); c_ry[q] = dsub(dmul(uy, ca), dmul(ux, sa));
            nbr[q] = j;
          }
          m += __popc(mask);
        }
        __syncwarp();
        const double grid = beh[11], ms = beh[12];
        const double lxa = dsub(vx, beh[3]), lxb = -beh[1], hxa = dadd(vx, beh[3]), hxb = beh[1];
        const double lya = dsub(vy, beh[3]), lyb = -beh[2], hya = dadd(vy, beh[3]), hyb = beh[2];
        const double lox = lxa > lxb ? lxa : lxb, hix = hxa < hxb ? hxa : hxb;
        const double loy = lya > lyb ? lya : lyb, hiy = hya < hyb ? hya : hyb;
        const int nx = world_rvo_count(lox, hix, grid), ny = world_rvo_count(loy, hiy, grid), nc = nx * ny;
        // pass 1: the closest candidate to v_des outside every cone
        double bkey = INFINITY;
        int bidx = INT_MAX;
        bool any = false;
        for (int k = lane; k < nc; k += 32) {
          const int kx = k / ny, ky = k - kx * ny;
          const double ux = dadd(lox, dmul((double)kx, grid)), uy = dadd(loy, dmul((double)ky, grid));
          if (__dsqrt_rn(ddot(ux, uy, ux, uy)) < ms) continue;
          any = true;
          bool out = true;
          for (int q = 0; q < m; ++q) {
            const double wx = dsub(ux, c_ax[q]), wy = dsub(uy, c_ay[q]);
            if (dcross(c_lx[q], c_ly[q], wx, wy) <= 0.0 && dcross(c_rx[q], c_ry[q], wx, wy) >= 0.0) { out = false; break; }
          }
          if (!out) continue;
          const double ex = dsub(ux, desx), ey = dsub(uy, desy), key = __dsqrt_rn(ddot(ex, ey, ex, ey));
          if (key < bkey) { bkey = key; bidx = k; }  // k ascends per lane: the lower index keeps a tie
        }
        if (__any_sync(0xffffffffu, bidx != INT_MAX)) {
          world_rvo_argmin(bkey, bidx);
        } else if (__any_sync(0xffffffffu, any)) {  // pass 2: every candidate is inside a cone -- the smallest penalty
          const double factor = beh[4];
          for (int k = lane; k < nc; k += 32) {
            const int kx = k / ny, ky = k - kx * ny;
            const double ux = dadd(lox, dmul((double)kx, grid)), uy = dadd(loy, dmul((double)ky, grid));
            if (__dsqrt_rn(ddot(ux, uy, ux, uy)) < ms) continue;
            double tmin = INFINITY;
            for (int q = 0; q < m; ++q) {
              const int j = nbr[q];
              const double tc = world_rvo_tc(dsub(s_cx[j], cx), dsub(s_cy[j], cy), dsub(ux, s_vx[j]), dsub(uy, s_vy[j]), dadd(ri, s_r[j]));
              tmin = tc < tmin ? tc : tmin;
            }
            const double ex = dsub(ux, desx), ey = dsub(uy, desy);
            const double pen = dadd(__ddiv_rn(factor, tmin), __dsqrt_rn(ddot(ex, ey, ex, ey)));
            if (pen < bkey || (pen == bkey && k < bidx)) { bkey = pen; bidx = k; }
          }
          world_rvo_argmin(bkey, bidx);
        }
        if (bidx != INT_MAX) {
          const int kx = bidx / ny, ky = bidx - kx * ny;
          nvx = dadd(lox, dmul((double)kx, grid)); nvy = dadd(loy, dmul((double)ky, grid));
        } else {
          nvx = vx; nvy = vy;
        }
        __syncwarp();  // the cone list is read by every lane before the next obstacle overwrites it
      }
      if (lane == 0) {
        double* row = prm.obs + (size_t)kWorldObsCols * o;
        row[2] = nvx; row[3] = nvy;
        rp.goal[2 * o] = gx; rp.goal[2 * o + 1] = gy;
        rp.draws[o] = draws;
      }
    }
  }
}

}  // namespace nb
