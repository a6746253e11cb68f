// Per-control-step work of InitialPath, batched over environments (SURVEY 8f "next" row 1): what neupan.forward does before
// PAN (neupan/neupan.py:114-121) -- check_arrive (neupan/blocks/initial_path.py:251-292, closest_point :166-183) and
// generate_nom_ref_state (:68-126, find_interaction_point / range_cir_seg :185-249, motion models :386-444).
//
// One thread per environment: the logic is a short sequential walk (T steps, a window of ind_range path points) with
// per-environment persistent state (curve_index, point_index, arrive_flag) and a MUTABLE path: the reference hands out numpy
// views of its path points and writes the aligned heading through them (initial_path.py:99,112) and wraps the heading of the
// last point in place (:191-192); entries of the returned reference trajectory that alias one stored point (the clamped tail
// of a curve) change together, and all of it persists across control steps.  The kernel reproduces that with write-through
// to the per-environment copy of the path in global memory and a read-back of the aliased entries after the T loop.
// Arithmetic in FP64 like numpy / math, float32 at the stores (np_to_tensor, neupan.py:123-126).
#pragma once
#include <cstdint>

namespace nb {

struct IpathParams {
  int B, T, kinematics, loop, ind_range, arrive_index_threshold;
  double dt, L, arrive_threshold, close_threshold, ref_speed;
  double* pts;                   // (P, 4): x, y, theta, gear -- mutable
  const int32_t* curve_begin;    // (C + 1) offsets into pts
  const int32_t* env_curve_begin;  // (B + 1) offsets into curve_begin
  const double* interval;        // (B) average point spacing of the env's whole path (cal_average_interval, :146-164)
  int32_t* curve_index;          // (B) persistent
  int32_t* point_index;          // (B) persistent
  int32_t* arrive_flag;          // (B) persistent
  const double* states;          // (B, 3)
  const float* cur_vel;          // (B, 2, T)
  float* nom_s;                  // (B, 3, T+1)
  float* nom_u;                  // (B, 2, T)
  float* ref_s;                  // (B, 3, T+1)
  float* ref_us;                 // (B, T)
  int32_t* arrived;              // (B): return value of check_arrive
  const int32_t* env_index;      // (B) kIndex: row b steps the path and persistent state env_index[b] (0 .. n_env - 1)
  int n_env;                     // kIndex: the environments the handle holds paths for
};

constexpr int kIpathMaxT = 64;
constexpr double kPi = 3.141592653589793;

// x @ y for two-element float64 vectors as numpy evaluates it (cblas_ddot of OpenBLAS on FMA hardware: the second product
// is fused into the accumulation, fma(x1, y1, round(x0 y0)); checked against numpy on 20,000 random pairs).  The
// circle / segment walk sits on a knife edge when the path spacing equals ref_speed * dt (intersection parameter t2 ~ 1), so the
// last bit of these dot products decides which segment's heading the reference point gets.
__device__ __forceinline__ double dot2(double x0, double x1, double y0, double y1) { return fma(x1, y1, __dmul_rn(x0, y0)); }

__device__ __forceinline__ double wrap_to_pi(double rad) {  // util.WrapToPi (neupan/util/__init__.py:98-120)
  while (rad > kPi) rad = rad - 2 * kPi;
  while (rad < -kPi) rad = rad + 2 * kPi;
  return rad;
}

// kIndex (nb_ipath_step_ex with an env_index): row b (states, cur_vel and the outputs) steps environment e = env_index[b] (its path,
// interval and persistent indices); an index outside 0 .. n_env - 1 gives row b an arrived flag and zero trajectories.  Without it,
// e = b.
template <bool kIndex>
__global__ void __launch_bounds__(64) ipath_step_kernel(const IpathParams prm) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= prm.B) return;
  const int T = prm.T, T1 = T + 1;
  const int e = kIndex ? prm.env_index[b] : b;
  if (kIndex && (e < 0 || e >= prm.n_env)) {
    prm.arrived[b] = 1;
    for (int i = 0; i < 3 * T1; ++i) { prm.nom_s[(size_t)b * 3 * T1 + i] = 0.f; prm.ref_s[(size_t)b * 3 * T1 + i] = 0.f; }
    for (int i = 0; i < 2 * T; ++i) prm.nom_u[(size_t)b * 2 * T + i] = 0.f;
    for (int t = 0; t < T; ++t) prm.ref_us[(size_t)b * T + t] = 0.f;
    return;
  }
  const double sx = prm.states[3 * b], sy = prm.states[3 * b + 1], sth = prm.states[3 * b + 2];
  const int c0 = prm.env_curve_begin[e], ncurves = prm.env_curve_begin[e + 1] - c0;
  int ci = prm.curve_index[e], pi = prm.point_index[e];
  int p0 = prm.curve_begin[c0 + ci], len = prm.curve_begin[c0 + ci + 1] - p0;
  double* P = prm.pts;
#define PX(i) P[4 * (size_t)(p0 + (i))]
#define PY(i) P[4 * (size_t)(p0 + (i)) + 1]
#define PTH(i) P[4 * (size_t)(p0 + (i)) + 2]
#define PG(i) P[4 * (size_t)(p0 + (i)) + 3]

  // ---- check_arrive (initial_path.py:251-292) -----------------------------------------------------------
  {  // closest_point (:166-183): window [point_index, point_index + ind_range), early exit below close_threshold
    double min_dis = __longlong_as_double(0x7ff0000000000000LL);
    const int start = pi > 0 ? pi : 0, end = min(pi + prm.ind_range, len);
    for (int i = start; i < end; ++i) {
      const double dx = sx - PX(i), dy = sy - PY(i);
      const double dis = sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
      if (dis < min_dis) {
        min_dis = dis;
        pi = i;
        if (dis < prm.close_threshold) break;
      }
    }
  }
  bool ret = false;
  {
    const double dx = sx - PX(len - 1), dy = sy - PY(len - 1);
    const bool arrive = sqrt(dot2(dx, dy, dx, dy)) < prm.arrive_threshold &&  // np.linalg.norm (:285-286)
                        pi >= len - prm.arrive_index_threshold - 2;  // check_curve_arrive (:282-290)
    if (arrive) {
      if (ci + 1 >= ncurves) {
        if (prm.loop) { ci = 0; pi = 0; }
        else { prm.arrive_flag[e] = 1; ret = true; }
      } else {
        ci += 1; pi = 0;
      }
      p0 = prm.curve_begin[c0 + ci];
      len = prm.curve_begin[c0 + ci + 1] - p0;
    }
  }
  prm.curve_index[e] = ci;
  prm.point_index[e] = pi;
  prm.arrived[b] = ret ? 1 : 0;
  float* ns = prm.nom_s + (size_t)b * 3 * T1;
  float* rs = prm.ref_s + (size_t)b * 3 * T1;
  float* nu = prm.nom_u + (size_t)b * 2 * T;
  float* ru = prm.ref_us + (size_t)b * T;
  const float* cv = prm.cur_vel + (size_t)b * 2 * T;
  for (int i = 0; i < 2 * T; ++i) nu[i] = cv[i];  // nom_u = cur_vel_array (:116)
  if (ret) {  // neupan.forward returns before generate_nom_ref_state (neupan.py:114-116)
    for (int i = 0; i < 3 * T1; ++i) { ns[i] = 0.f; rs[i] = 0.f; }
    for (int t = 0; t < T; ++t) ru[t] = 0.f;
    return;
  }

  // ---- generate_nom_ref_state (initial_path.py:68-126) -------------------------------------------------
  double rx = PX(pi), ry = PY(pi), rth = PTH(pi);  // ref_state = cur_point[0:3].copy()
  int alias = -1;                                  // >= 0: ref_state is a view of path point `alias`
  int ref_index = pi;
  double px_ = sx, py_ = sy, pth = sth;            // pre_state
  const double gear0 = PG(pi);
  const double fwd = prm.ref_speed * prm.dt;
  const double interval = prm.interval[e];
  int alias_of[kIpathMaxT];
  ns[0] = (float)px_; ns[T1] = (float)py_; ns[2 * T1] = (float)pth;
  rs[0] = (float)rx; rs[T1] = (float)ry; rs[2 * T1] = (float)rth;
  for (int t = 0; t < T; ++t) {
    const double v = (double)cv[t], w = (double)cv[T + t];
    if (prm.kinematics == 1) {  // acker (:401-415)
      const double d0 = v * cos(pth), d1 = v * sin(pth), d2 = v * tan(w) / prm.L;
      px_ = __dadd_rn(px_, __dmul_rn(d0, prm.dt)); py_ = __dadd_rn(py_, __dmul_rn(d1, prm.dt)); pth = __dadd_rn(pth, __dmul_rn(d2, prm.dt));
    } else if (prm.kinematics == 0) {  // diff (:417-430)
      const double d0 = v * cos(pth), d1 = v * sin(pth);
      px_ = __dadd_rn(px_, __dmul_rn(d0, prm.dt)); py_ = __dadd_rn(py_, __dmul_rn(d1, prm.dt)); pth = __dadd_rn(pth, __dmul_rn(w, prm.dt));
    } else {  // omni (:432-444)
      const double vx = v * cos(w), vy = v * sin(w);
      px_ = __dadd_rn(px_, __dmul_rn(prm.dt, vx)); py_ = __dadd_rn(py_, __dmul_rn(prm.dt, vy)); pth = __dadd_rn(pth, __dmul_rn(prm.dt, 0.0));
    }
    ns[t + 1] = (float)px_; ns[T1 + t + 1] = (float)py_; ns[2 * T1 + t + 1] = (float)pth;
    double gear = gear0;
    if (fwd >= interval) {  // jump by whole path points (:91-101)
      ref_index = ref_index + (int)(fwd / interval);
      if (ref_index > len - 1) { ref_index = len - 1; gear = 0.0; }
      alias = ref_index;
    } else {  // circle / segment intersection walk (:103-109, find_interaction_point :185-215)
      const double cx = alias >= 0 ? PX(alias) : rx, cy = alias >= 0 ? PY(alias) : ry;
      for (;;) {
        if (ref_index > len - 2) {
          PTH(len - 1) = wrap_to_pi(PTH(len - 1));  // in place (:191-192)
          alias = len - 1;
          break;
        }
        const double ax = PX(ref_index), ay = PY(ref_index), bx = PX(ref_index + 1), by = PY(ref_index + 1);
        const double dx = bx - ax, dy = by - ay;
        bool hit = false;
        if (sqrt(dot2(dx, dy, dx, dy)) != 0.0) {  // range_cir_seg (:217-249)
          const double fx = ax - cx, fy = ay - cy;
          const double a = dot2(dx, dy, dx, dy);                       // d @ d
          const double bq = __dmul_rn(2.0, dot2(fx, fy, dx, dy));      // 2 * f @ d  (= (2 f) @ d: scaling by two is exact)
          const double c = dot2(fx, fy, fx, fy) - __dmul_rn(fwd, fwd);  // f @ f - r**2
          const double disc = __dadd_rn(__dmul_rn(bq, bq), -__dmul_rn(__dmul_rn(4.0, a), c));
          if (!(disc < 0)) {
            const double t2 = (-bq + sqrt(disc)) / __dmul_rn(2.0, a);
            if (t2 >= 0 && t2 <= 1) {
              rx = __dadd_rn(ax, __dmul_rn(t2, dx));
              ry = __dadd_rn(ay, __dmul_rn(t2, dy));
              const double diff = wrap_to_pi(PTH(ref_index + 1) - PTH(ref_index));
              rth = wrap_to_pi(PTH(ref_index) + diff / 2);
              alias = -1;
              hit = true;
            }
          }
        }
        if (hit) break;
        ref_index += 1;
      }
      if (ref_index > len - 1) gear = 0.0;
    }
    if (alias >= 0) {  // heading aligned to the predicted state, written THROUGH the view (:111-112)
      const double th = PTH(alias);
      PTH(alias) = pth + wrap_to_pi(th - pth);
    } else {
      rth = pth + wrap_to_pi(rth - pth);
      rs[t + 1] = (float)rx; rs[T1 + t + 1] = (float)ry; rs[2 * T1 + t + 1] = (float)rth;
    }
    alias_of[t] = alias;
    ru[t] = (float)(gear * prm.ref_speed);  // ref_us = gear_array * ref_speed (:124)
  }
  for (int t = 0; t < T; ++t) {  // np.hstack after the loop: aliased entries show the final content of the path point
    const int q = alias_of[t];
    if (q >= 0) { rs[t + 1] = (float)PX(q); rs[T1 + t + 1] = (float)PY(q); rs[2 * T1 + t + 1] = (float)PTH(q); }
  }
#undef PX
#undef PY
#undef PTH
#undef PG
}

}  // namespace nb
