// Batched 2-D world for closed-loop runs of B planners: what IR-SIM does between two planner calls (example/run_exp.py:27-56,
// env.get_lidar_scan / env.step / env.done), for B environments at once and without leaving the device.
//
// Scene: per environment a ragged list of obstacles -- circles (centre, radius), convex polygons (3..8 vertices) and outlines (any
// simple polygon of 3..16 vertices, convex or not; kind 1), vertices stored relative to the centre so that motion only moves the
// centre -- each with a constant world-frame velocity, an axis-aligned rectangle in which moving obstacles bounce, and K robots
// (1 <= K <= 16, nb_world_set_fleet; one without a fleet) of the planner's robot polygon, each with its goal.  Robot k of
// environment b is row n = b K + k of every per-robot array.
//
//   world_scan_kernel        one CTA per environment (grid-stride): the environment's circles and polygon edges (convex and outline
//                            alike) and, with K > 1, the K robot bodies (edges tagged with their owner) are staged in shared memory in
//                            world coordinates with each robot's sensor pose, then one thread per beam of the K R beams finds the first
//                            boundary crossing with t > 0; a beam skips its own robot's edges
//   world_step_kernel        K = 1: one warp per environment: obstacles move (reflecting at the rectangle), the robot integrates its
//                            action unless it has collided, then the exact clearance robot polygon <-> every obstacle, reduced over the warp
//   world_fleet_step_kernel  K > 1: one CTA per environment: the robots integrate (Jacobi: from the states at the start of the step),
//                            their world vertices and velocities go to shared memory and the obstacles move; after a barrier one warp per
//                            robot takes the clearance to every obstacle (world_step_kernel's branches) and to every other robot
//                            (convex-convex, symmetric bit for bit), then a warp min
//
// Several robots (this project's reading of an IR-SIM world whose robot: section lists several robots): a beam also tests the bodies
// of the other K - 1 robots (the robot polygon at their current state), never its own; a robot hit reports index O_b + j (O_b the
// environment's obstacle count), so at equal t an obstacle wins, and the world-frame velocity of the action that robot integrated in
// the last step (0 before the first step and once it has collided; translation only, omega x r left out).  collided is sticky and
// freezes a robot, which stays in the scene; arrived is sticky and an arrived robot stays in the scene.
//
// All arithmetic is FP64 with explicit rounding (__dmul_rn / __dadd_rn / __dsub_rn: no FMA contraction), so that oracle/world.py,
// which performs the same operations in the same order in numpy, agrees to the last bit wherever the inputs agree (the only
// differences come from CUDA's sin / cos / tan vs libm).
#pragma once
#include <cstdint>

namespace nb {

constexpr int kWorldMaxObstacles = 256;  // per environment (staged in shared memory by the scan kernel)
constexpr int kWorldMaxVertices = 8;     // per convex polygon (obstacles and the robot)
constexpr int kWorldMaxOutlineVertices = 16;
constexpr int kWorldMaxEdges = 2048;     // polygon edges (convex and outline) per environment, staged in shared memory by the scan
constexpr int kWorldObsCols = 5;         // obstacle row: cx, cy, vx, vy, radius (radius unused for polygons)
constexpr int kWorldEnvCols = 10;        // env row: xmin, ymin, xmax, ymax, start x, y, theta, goal x, y, goal threshold
constexpr int kWorldStepWarps = 4;
constexpr int kWorldMaxFleet = 16;       // robots per environment
constexpr int kWorldFleetWarps = 8;      // world_fleet_step_kernel: at most 8 warps per CTA, warp w takes robots w, w + 8

struct WorldParams {
  int B, R, kinematics, robot_nv;
  double dt, L, range_max;
  double off_x, off_y, off_th;
  double robot_v[2 * kWorldMaxVertices];  // robot polygon in its own frame: x0, y0, x1, y1, ...
  const double* beam_cs;                  // (R, 2) cos, sin of a_i = linspace(angle_min, angle_max, R)[i] (libm, on the host)
  const int32_t* obs_begin;               // (B + 1) offsets into the obstacle rows
  const int32_t* vert_begin;              // (O + 1) offsets into vertices; an empty range is a circle
  const int32_t* slot;                    // (O) circle: rank among the env's circles; polygon: index of its first edge in the env
  const int32_t* counts;                  // (B, 2) circles, polygon edges of the environment
  const int32_t* kind;                    // (O) 0: circle or convex polygon, 1: outline
  const double* vertices;                 // (V, 2) relative to the obstacle's centre
  const double* env;                      // (B, kWorldEnvCols)
  double* obs;                            // (O, kWorldObsCols) -- centres and velocities change
  double* states;                         // (B, 3) x, y, theta
  int32_t* collided;                      // (B) sticky
  int32_t* arrived;                       // (B) sticky
  int K;                                  // robots per environment: states (B K, 3), collided and arrived (B K)
  const double* fgoal;                    // (B K, 3) goal x, y, threshold of every robot (K > 1)
  double* fvel;                           // (B K, 2) world-frame velocity of each robot's last step (K > 1)
};

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ddot(double ax, double ay, double bx, double by) { return dadd(dmul(ax, bx), dmul(ay, by)); }
__device__ __forceinline__ double dcross(double ax, double ay, double bx, double by) { return dsub(dmul(ax, by), dmul(ay, bx)); }

// ---- lidar ----------------------------------------------------------------------------------------------------------------

// Beam i of robot k leaves that robot's sensor at world angle (theta + off_th) + a_i, a_i = linspace(angle_min, angle_max, R)[i] --
// the convention nb_scan_to_points inverts.  Its direction is evaluated as the rotation of (cos a_i, sin a_i) by the sensor heading:
// no trigonometry per beam (and none of the argument-reduction slow path, whose call would spill the beam loop's registers); the
// sensor poses are computed once per environment and staged in shared memory.  range = the smallest t > 0 at which the ray crosses an
// obstacle boundary or, with K > 1, the body of another robot of the environment (a sensor inside an obstacle or another robot sees
// the exit crossing); t >= range_max or no crossing is a miss: range_max, velocity 0, hit -1.  Equal t: the lower index wins
// (obstacles 0..O_b - 1, then robot j as O_b + j), so the result does not depend on the order of the tests.
__global__ void __launch_bounds__(256) world_scan_kernel(const WorldParams prm, int max_circ, int max_edges, float* __restrict__ ranges,
                                                         float* __restrict__ velocity, int32_t* __restrict__ hit) {
  extern __shared__ double wsm[];
  __shared__ double s_sx[kWorldMaxFleet], s_sy[kWorldMaxFleet], s_hc[kWorldMaxFleet], s_hs[kWorldMaxFleet];  // sensor poses
  const int K = prm.K, nr = prm.robot_nv;
  const int nre = K > 1 ? K * nr : 0;  // robot edges: a single robot stages none
  double* r_ax = wsm;
  double* r_ay = r_ax + nre;
  double* r_bx = r_ay + nre;
  double* r_by = r_bx + nre;
  double* c_x = r_by + nre;
  double* c_y = c_x + max_circ;
  double* c_r = c_y + max_circ;
  double* e_ax = c_r + max_circ;
  double* e_ay = e_ax + max_edges;
  double* e_bx = e_ay + max_edges;
  double* e_by = e_bx + max_edges;
  int32_t* c_id = reinterpret_cast<int32_t*>(e_by + max_edges);
  int32_t* e_id = c_id + max_circ;
  int32_t* r_id = e_id + max_edges;  // owner of each robot edge
  const int R = prm.R;
  for (int b = blockIdx.x; b < prm.B; b += gridDim.x) {
    const int o0 = prm.obs_begin[b], o1 = prm.obs_begin[b + 1];
    const int nc = prm.counts[2 * b], ne = prm.counts[2 * b + 1];
    __syncthreads();  // the previous environment's beams are done with the shared lists
    for (int o = o0 + (int)threadIdx.x; o < o1; o += blockDim.x) {
      const double cx = prm.obs[kWorldObsCols * o], cy = prm.obs[kWorldObsCols * o + 1];
      const int v0 = prm.vert_begin[o], nv = prm.vert_begin[o + 1] - v0, s = prm.slot[o];
      if (nv == 0) {
        c_x[s] = cx; c_y[s] = cy; c_r[s] = prm.obs[kWorldObsCols * o + 4]; c_id[s] = o - o0;
      } else {
        for (int k = 0; k < nv; ++k) {
          const int k1 = k + 1 < nv ? k + 1 : 0;
          e_ax[s + k] = dadd(cx, prm.vertices[2 * (v0 + k)]);
          e_ay[s + k] = dadd(cy, prm.vertices[2 * (v0 + k) + 1]);
          e_bx[s + k] = dadd(cx, prm.vertices[2 * (v0 + k1)]);
          e_by[s + k] = dadd(cy, prm.vertices[2 * (v0 + k1) + 1]);
          e_id[s + k] = o - o0;
        }
      }
    }
    for (int k = threadIdx.x; k < K; k += blockDim.x) {  // robot k: sensor pose, and with K > 1 its body (the step kernel's vertices)
      const size_t n = (size_t)b * K + k;
      const double x = prm.states[3 * n], y = prm.states[3 * n + 1], th = prm.states[3 * n + 2];
      double sn, cs;
      sincos(th, &sn, &cs);
      s_sx[k] = dadd(x, dsub(dmul(cs, prm.off_x), dmul(sn, prm.off_y)));  // sensor position: robot pose applied to scan_offset
      s_sy[k] = dadd(y, dadd(dmul(sn, prm.off_x), dmul(cs, prm.off_y)));
      double hs, hc;
      sincos(dadd(th, prm.off_th), &hs, &hc);
      s_hc[k] = hc; s_hs[k] = hs;
      if (nre) {
        double vx[kWorldMaxVertices], vy[kWorldMaxVertices];
#pragma unroll
        for (int v = 0; v < kWorldMaxVertices; ++v) {  // constant indices: the parameter array and vx / vy stay in registers
          const double px = prm.robot_v[2 * v], py = prm.robot_v[2 * v + 1];
          vx[v] = dadd(x, dsub(dmul(cs, px), dmul(sn, py)));
          vy[v] = dadd(y, dadd(dmul(sn, px), dmul(cs, py)));
        }
#pragma unroll
        for (int v = 0; v < kWorldMaxVertices; ++v) {
          if (v < nr) {
            const int e = k * nr + v;
            const bool last = v + 1 == nr;
            r_ax[e] = vx[v]; r_ay[e] = vy[v];
            r_bx[e] = last ? vx[0] : vx[v + 1 < kWorldMaxVertices ? v + 1 : 0];
            r_by[e] = last ? vy[0] : vy[v + 1 < kWorldMaxVertices ? v + 1 : 0];
            r_id[e] = k;
          }
        }
      }
    }
    __syncthreads();
    const int nobs = o1 - o0;
    for (int q = threadIdx.x; q < K * R; q += blockDim.x) {
      const int k = K == 1 ? 0 : q / R, i = q - k * R;
      const double sx = s_sx[k], sy = s_sy[k], hc = s_hc[k], hs = s_hs[k];
      const double ca = prm.beam_cs[2 * i], sa = prm.beam_cs[2 * i + 1];  // the beam's direction: the sensor heading rotated by a_i
      const double dx = dsub(dmul(hc, ca), dmul(hs, sa)), dy = dadd(dmul(hs, ca), dmul(hc, sa));
      double best = INFINITY;
      int bid = 0x7fffffff;
      for (int j = 0; j < nc; ++j) {  // |s + t d - c|^2 = r^2 with |d| = 1: t = -b -+ sqrt(b^2 - c)
        const double fx = dsub(sx, c_x[j]), fy = dsub(sy, c_y[j]);
        const double bq = ddot(fx, fy, dx, dy);
        const double cq = dsub(ddot(fx, fy, fx, fy), dmul(c_r[j], c_r[j]));
        const double disc = dsub(dmul(bq, bq), cq);
        if (disc >= 0.0) {
          const double sq = sqrt(disc);
          double t = dsub(-bq, sq);
          if (!(t > 0.0)) t = dadd(-bq, sq);
          if (t > 0.0 && (t < best || (t == best && c_id[j] < bid))) { best = t; bid = c_id[j]; }
        }
      }
      for (int j = 0; j < ne; ++j) {  // s + t d = a + u e:  t = (w x e) / (d x e), u = (w x d) / (d x e), w = a - s
        const double ex = dsub(e_bx[j], e_ax[j]), ey = dsub(e_by[j], e_ay[j]);
        const double den = dcross(dx, dy, ex, ey);
        if (den != 0.0) {
          const double wx = dsub(e_ax[j], sx), wy = dsub(e_ay[j], sy);
          const double t = dcross(wx, wy, ex, ey) / den, u = dcross(wx, wy, dx, dy) / den;
          if (u >= 0.0 && u <= 1.0 && t > 0.0 && (t < best || (t == best && e_id[j] < bid))) { best = t; bid = e_id[j]; }
        }
      }
      for (int j = 0; j < nre; ++j) {  // the other robots' bodies, the same edge test
        if (r_id[j] == k) continue;
        const double ex = dsub(r_bx[j], r_ax[j]), ey = dsub(r_by[j], r_ay[j]);
        const double den = dcross(dx, dy, ex, ey);
        if (den != 0.0) {
          const double wx = dsub(r_ax[j], sx), wy = dsub(r_ay[j], sy);
          const double t = dcross(wx, wy, ex, ey) / den, u = dcross(wx, wy, dx, dy) / den;
          const int id = nobs + r_id[j];
          if (u >= 0.0 && u <= 1.0 && t > 0.0 && (t < best || (t == best && id < bid))) { best = t; bid = id; }
        }
      }
      if (!(best < prm.range_max)) { best = prm.range_max; bid = -1; }
      const size_t n = (size_t)b * K + k;
      ranges[n * R + i] = (float)best;
      if (velocity) {
        float vx = 0.f, vy = 0.f;
        if (bid >= nobs) {
          const double* fv = prm.fvel + 2 * ((size_t)b * K + (bid - nobs));
          vx = (float)fv[0]; vy = (float)fv[1];
        } else if (bid >= 0) {
          const double* row = prm.obs + (size_t)kWorldObsCols * (o0 + bid);
          vx = (float)row[2]; vy = (float)row[3];
        }
        velocity[n * 2 * R + i] = vx;
        velocity[n * 2 * R + R + i] = vy;
      }
      if (hit) hit[n * R + i] = bid;
    }
  }
}

// ---- clearance ------------------------------------------------------------------------------------------------------------

// distance from p to the segment a-b (a != b)
__device__ __forceinline__ double world_seg_dist(double px, double py, double ax, double ay, double bx, double by) {
  const double ex = dsub(bx, ax), ey = dsub(by, ay), wx = dsub(px, ax), wy = dsub(py, ay);
  double t = ddot(wx, wy, ex, ey) / ddot(ex, ey, ex, ey);
  t = t < 0.0 ? 0.0 : (t > 1.0 ? 1.0 : t);
  const double qx = dsub(wx, dmul(t, ex)), qy = dsub(wy, dmul(t, ey));
  return sqrt(ddot(qx, qy, qx, qy));
}

// Vertex accessors of the two polygons of a clearance test: the obstacle's world vertex k (k < nv) is its centre plus the stored
// offset; the robot's world vertices sit in shared memory.
struct WorldPoly {
  const double* rel;  // nv rows of (dx, dy)
  double cx, cy;
  int nv;
  __device__ __forceinline__ double vx(int k) const { return dadd(cx, rel[2 * k]); }
  __device__ __forceinline__ double vy(int k) const { return dadd(cy, rel[2 * k + 1]); }
};
struct WorldRobot {
  const double *x, *y;  // world vertices
  int nv;
  __device__ __forceinline__ double vx(int k) const { return x[k]; }
  __device__ __forceinline__ double vy(int k) const { return y[k]; }
};

// Does an edge normal of convex polygon A separate A from B?  Projections onto n = (-e_y, e_x) of every edge e of A.
template <class PA, class PB>
__device__ __forceinline__ bool world_sat_separates(const PA& a, const PB& bp) {
  for (int k = 0; k < a.nv; ++k) {
    const int k1 = k + 1 < a.nv ? k + 1 : 0;
    const double nx = -dsub(a.vy(k1), a.vy(k)), ny = dsub(a.vx(k1), a.vx(k));
    double amin = INFINITY, amax = -INFINITY, bmin = INFINITY, bmax = -INFINITY;
    for (int i = 0; i < a.nv; ++i) {
      const double p = ddot(nx, ny, a.vx(i), a.vy(i));
      amin = fmin(amin, p); amax = fmax(amax, p);
    }
    for (int i = 0; i < bp.nv; ++i) {
      const double p = ddot(nx, ny, bp.vx(i), bp.vy(i));
      bmin = fmin(bmin, p); bmax = fmax(bmax, p);
    }
    if (amax < bmin || bmax < amin) return true;
  }
  return false;
}

// p lies in the bounding box of the segment a-b (with a zero orientation: p lies on the closed segment)
__device__ __forceinline__ bool world_in_box(double ax, double ay, double bx, double by, double px, double py) {
  return fmin(ax, bx) <= px && px <= fmax(ax, bx) && fmin(ay, by) <= py && py <= fmax(ay, by);
}

// Do the closed segments p-q and a-b intersect or touch?  Orientation tests; a zero orientation (collinear, or an endpoint on the
// other segment's line) counts when that endpoint lies within the other segment.
__device__ __forceinline__ bool world_segs_meet(double px, double py, double qx, double qy, double ax, double ay, double bx, double by) {
  const double ex = dsub(bx, ax), ey = dsub(by, ay), fx = dsub(qx, px), fy = dsub(qy, py);
  const double d1 = dcross(ex, ey, dsub(px, ax), dsub(py, ay)), d2 = dcross(ex, ey, dsub(qx, ax), dsub(qy, ay));
  const double d3 = dcross(fx, fy, dsub(ax, px), dsub(ay, py)), d4 = dcross(fx, fy, dsub(bx, px), dsub(by, py));
  if (((d1 > 0.0 && d2 < 0.0) || (d1 < 0.0 && d2 > 0.0)) && ((d3 > 0.0 && d4 < 0.0) || (d3 < 0.0 && d4 > 0.0))) return true;
  return (d1 == 0.0 && world_in_box(ax, ay, bx, by, px, py)) || (d2 == 0.0 && world_in_box(ax, ay, bx, by, qx, qy)) ||
         (d3 == 0.0 && world_in_box(px, py, qx, qy, ax, ay)) || (d4 == 0.0 && world_in_box(px, py, qx, qy, bx, by));
}

// Robot (convex) <-> outline (any simple polygon): 0 when they overlap -- an outline edge meets a robot edge, robot vertex 0 lies
// inside the outline, or outline vertex 0 lies inside the robot (the circle branch's sign test) -- else the smallest vertex-edge
// distance both ways, in the convex branch's order (so a convex polygon given as an outline gets the same distance bit for bit).
// The even-odd test of robot vertex 0 shares the edge loop of the segment tests (separate loops spill): an outline edge that
// straddles the horizontal line through the vertex toggles it when it crosses that line to the vertex's right, which is the sign
// of the cross product edge x (vertex - edge start) -- no division.
__device__ __forceinline__ double world_outline_clearance(const WorldPoly& op, const double* rx, const double* ry, int nr) {
  bool in = false;
  for (int k = 0; k < op.nv; ++k) {
    const int k1 = k + 1 < op.nv ? k + 1 : 0;
    const double ax = op.vx(k), ay = op.vy(k), bx = op.vx(k1), by = op.vy(k1);
    for (int i = 0; i < nr; ++i) {
      const int i1 = i + 1 < nr ? i + 1 : 0;
      if (world_segs_meet(rx[i], ry[i], rx[i1], ry[i1], ax, ay, bx, by)) return 0.0;
    }
    if ((ay > ry[0]) != (by > ry[0])) {
      const double c = dcross(dsub(bx, ax), dsub(by, ay), dsub(rx[0], ax), dsub(ry[0], ay));
      if (by > ay ? c > 0.0 : c < 0.0) in = !in;
    }
  }
  if (in) return 0.0;
  {
    const double px = op.vx(0), py = op.vy(0);
    bool pos = false, neg = false;
    for (int k = 0; k < nr; ++k) {
      const int k1 = k + 1 < nr ? k + 1 : 0;
      const double cr = dcross(dsub(rx[k1], rx[k]), dsub(ry[k1], ry[k]), dsub(px, rx[k]), dsub(py, ry[k]));
      pos |= cr > 0.0; neg |= cr < 0.0;
    }
    if (!(pos && neg)) return 0.0;
  }
  double d = INFINITY;
  for (int k = 0; k < op.nv; ++k) {
    const int k1 = k + 1 < op.nv ? k + 1 : 0;
    const double ax = op.vx(k), ay = op.vy(k), bx = op.vx(k1), by = op.vy(k1);
    for (int i = 0; i < nr; ++i) d = fmin(d, world_seg_dist(rx[i], ry[i], ax, ay, bx, by));
  }
  for (int k = 0; k < nr; ++k) {
    const int k1 = k + 1 < nr ? k + 1 : 0;
    for (int i = 0; i < op.nv; ++i) d = fmin(d, world_seg_dist(op.vx(i), op.vy(i), rx[k], ry[k], rx[k1], ry[k1]));
  }
  return d;
}

// ---- step ----------------------------------------------------------------------------------------------------------------

// One step of the motion models from (x, y, th); (vx, vy) is the world-frame translation rate it used (diff / acker v (cos th, sin th)
// with the heading before the step, omni (vx, vy)).
__device__ __forceinline__ void world_integrate(const WorldParams& prm, double a0, double a1, double& x, double& y, double& th, double& vx,
                                                double& vy) {
  double dth;
  if (prm.kinematics == 2) {  // omni: the (vx, vy) PlannerBatch returns
    vx = a0; vy = a1; dth = 0.0;
  } else {
    double sn, cs;
    sincos(th, &sn, &cs);
    vx = dmul(a0, cs); vy = dmul(a0, sn);
    dth = prm.kinematics == 1 ? dmul(a0, tan(a1)) / prm.L : a1;  // acker: v tan(phi) / L; diff: omega
  }
  x = dadd(x, dmul(vx, prm.dt)); y = dadd(y, dmul(vy, prm.dt)); th = dadd(th, dmul(dth, prm.dt));
}

// Obstacle o moves by v dt; a moving centre that left the rectangle is mirrored back and its velocity component reversed.  Writes
// the row and returns the new centre.
__device__ __forceinline__ void world_move_obstacle(const WorldParams& prm, const double* env, int o, double& cx, double& cy) {
  double* row = prm.obs + (size_t)kWorldObsCols * o;
  double vx = row[2], vy = row[3];
  cx = dadd(row[0], dmul(vx, prm.dt));
  cy = dadd(row[1], dmul(vy, prm.dt));
  if (vx != 0.0) {
    if (cx < env[0]) { cx = dsub(dmul(2.0, env[0]), cx); vx = -vx; }
    else if (cx > env[2]) { cx = dsub(dmul(2.0, env[2]), cx); vx = -vx; }
  }
  if (vy != 0.0) {
    if (cy < env[1]) { cy = dsub(dmul(2.0, env[1]), cy); vy = -vy; }
    else if (cy > env[3]) { cy = dsub(dmul(2.0, env[3]), cy); vy = -vy; }
  }
  row[0] = cx; row[1] = cy; row[2] = vx; row[3] = vy;
}

// Clearance of the robot polygon (world vertices rx, ry) to obstacle o centred at (cx, cy), not yet clamped at 0.
__device__ __forceinline__ double world_obstacle_clearance(const WorldParams& prm, int o, double cx, double cy, const double* rx,
                                                           const double* ry, int nr) {
  const int v0 = prm.vert_begin[o], nv = prm.vert_begin[o + 1] - v0;
  if (nv == 0) {  // circle: distance from the centre to the robot polygon - r
    bool pos = false, neg = false;
    double d = INFINITY;
    for (int k = 0; k < nr; ++k) {
      const int k1 = k + 1 < nr ? k + 1 : 0;
      const double cr = dcross(dsub(rx[k1], rx[k]), dsub(ry[k1], ry[k]), dsub(cx, rx[k]), dsub(cy, ry[k]));
      pos |= cr > 0.0; neg |= cr < 0.0;
      d = fmin(d, world_seg_dist(cx, cy, rx[k], ry[k], rx[k1], ry[k1]));
    }
    return (pos && neg) ? dsub(d, prm.obs[(size_t)kWorldObsCols * o + 4]) : 0.0;  // centre inside the robot: overlap
  }
  if (prm.kind[o] != 0) return world_outline_clearance(WorldPoly{prm.vertices + 2 * (size_t)v0, cx, cy, nv}, rx, ry, nr);
  // convex polygon: 0 unless an edge normal separates them, then the smallest vertex-edge distance
  const WorldPoly op{prm.vertices + 2 * (size_t)v0, cx, cy, nv};
  const WorldRobot rp{rx, ry, nr};
  if (!(world_sat_separates(rp, op) || world_sat_separates(op, rp))) return 0.0;
  double d = INFINITY;
  for (int k = 0; k < nv; ++k) {
    const int k1 = k + 1 < nv ? k + 1 : 0;
    const double ax = op.vx(k), ay = op.vy(k), bx = op.vx(k1), by = op.vy(k1);
    for (int i = 0; i < nr; ++i) d = fmin(d, world_seg_dist(rx[i], ry[i], ax, ay, bx, by));
  }
  for (int k = 0; k < nr; ++k) {
    const int k1 = k + 1 < nr ? k + 1 : 0;
    for (int i = 0; i < nv; ++i) d = fmin(d, world_seg_dist(op.vx(i), op.vy(i), rx[k], ry[k], rx[k1], ry[k1]));
  }
  return d;
}

// Robot <-> robot (both convex): 0 unless an edge normal of either separates them (both SAT orders), else the smallest vertex-edge
// distance both ways.  Swapping a and b evaluates the same tests and distances and reduces them with fmin, so the result is
// symmetric bit for bit: two robots that touch collide in the same step.
__device__ __forceinline__ double world_robot_clearance(const WorldRobot& a, const WorldRobot& b) {
  if (!(world_sat_separates(a, b) || world_sat_separates(b, a))) return 0.0;
  double d = INFINITY;
  for (int k = 0; k < b.nv; ++k) {
    const int k1 = k + 1 < b.nv ? k + 1 : 0;
    for (int i = 0; i < a.nv; ++i) d = fmin(d, world_seg_dist(a.x[i], a.y[i], b.x[k], b.y[k], b.x[k1], b.y[k1]));
  }
  for (int k = 0; k < a.nv; ++k) {
    const int k1 = k + 1 < a.nv ? k + 1 : 0;
    for (int i = 0; i < b.nv; ++i) d = fmin(d, world_seg_dist(b.x[i], b.y[i], a.x[k], a.y[k], a.x[k1], a.y[k1]));
  }
  return d;
}

__global__ void __launch_bounds__(32 * kWorldStepWarps) world_step_kernel(const WorldParams prm, const float* __restrict__ action,
                                                                         int32_t* __restrict__ out_collided, int32_t* __restrict__ out_arrived,
                                                                         float* __restrict__ clearance) {
  __shared__ double rob[kWorldStepWarps][2][kWorldMaxVertices];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int b = blockIdx.x * kWorldStepWarps + w;
  if (b >= prm.B) return;  // whole warps leave together
  double* rx = rob[w][0];
  double* ry = rob[w][1];
  const double* env = prm.env + (size_t)kWorldEnvCols * b;
  // robot: every lane integrates the same state (no shuffles needed later); a collided robot stays where it is
  double x = prm.states[3 * b], y = prm.states[3 * b + 1], th = prm.states[3 * b + 2];
  const bool was_collided = prm.collided[b] != 0;
  if (!was_collided) {
    double vx, vy;
    world_integrate(prm, (double)action[2 * b], (double)action[2 * b + 1], x, y, th, vx, vy);
  }
  // everything that needs the robot's state is done before the obstacle loop, which keeps few values live across its divisions
  const double gx = dsub(x, env[7]), gy = dsub(y, env[8]);
  const int arr = (prm.arrived[b] != 0 || sqrt(ddot(gx, gy, gx, gy)) < env[9]) ? 1 : 0;
  {
    double sn, cs;
    sincos(th, &sn, &cs);
    double px = 0.0, py = 0.0;
#pragma unroll
    for (int k = 0; k < kWorldMaxVertices; ++k)  // constant indices: a kernel-parameter array indexed by lane would go to local memory
      if (lane == k) { px = prm.robot_v[2 * k]; py = prm.robot_v[2 * k + 1]; }
    if (lane < prm.robot_nv) {
      rx[lane] = dadd(x, dsub(dmul(cs, px), dmul(sn, py)));
      ry[lane] = dadd(y, dadd(dmul(sn, px), dmul(cs, py)));
    }
  }
  __syncwarp();  // the robot's vertices are published, and every lane has read the old state before lane 0 overwrites it
  if (lane == 0) { prm.states[3 * b] = x; prm.states[3 * b + 1] = y; prm.states[3 * b + 2] = th; }
  const int nr = prm.robot_nv;
  double best = INFINITY;
  for (int o = prm.obs_begin[b] + lane; o < prm.obs_begin[b + 1]; o += 32) {
    double cx, cy;
    world_move_obstacle(prm, env, o, cx, cy);
    const double c = world_obstacle_clearance(prm, o, cx, cy, rx, ry, nr);
    best = fmin(best, c > 0.0 ? c : 0.0);
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) best = fmin(best, __shfl_xor_sync(0xffffffffu, best, m));
  if (lane == 0) {
    const int col = (was_collided || best <= 0.0) ? 1 : 0;
    prm.collided[b] = col; prm.arrived[b] = arr;
    if (out_collided) out_collided[b] = col;
    if (out_arrived) out_arrived[b] = arr;
    if (clearance) clearance[b] = (float)best;
  }
}

// K > 1 robots per environment, one CTA of 32 min(K, 8) threads per environment (grid = B).  Phase 1: thread k integrates robot k
// from the state at the start of the step (unless it has collided), writes its state, arrival flag, world vertices and velocity; every
// thread moves obstacles.  Phase 2, after the barrier: one warp per robot (warp w takes robots w, w + 8; a 512-thread CTA would cap
// the registers at 128 and spill) computes its clearance to every obstacle (lanes over the obstacles, the branches of
// world_step_kernel) and to every other robot (lane j), a warp min, and lane 0 writes the collision flag, the clearance and the
// velocity the scan reports for the robot (0 once collided).
__global__ void __launch_bounds__(32 * kWorldFleetWarps) world_fleet_step_kernel(const WorldParams prm, const float* __restrict__ action,
                                                                              int32_t* __restrict__ out_collided, int32_t* __restrict__ out_arrived,
                                                                              float* __restrict__ clearance) {
  __shared__ double f_x[kWorldMaxFleet][kWorldMaxVertices], f_y[kWorldMaxFleet][kWorldMaxVertices];
  __shared__ double f_v[kWorldMaxFleet][2];
  const int K = prm.K, nr = prm.robot_nv, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int b = blockIdx.x;  // grid = B
  {
    const double* env = prm.env + (size_t)kWorldEnvCols * b;
    const int o0 = prm.obs_begin[b], o1 = prm.obs_begin[b + 1];
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
      const size_t n = (size_t)b * K + k;
      double x = prm.states[3 * n], y = prm.states[3 * n + 1], th = prm.states[3 * n + 2];
      double vx = 0.0, vy = 0.0;
      if (prm.collided[n] == 0) world_integrate(prm, (double)action[2 * n], (double)action[2 * n + 1], x, y, th, vx, vy);
      prm.states[3 * n] = x; prm.states[3 * n + 1] = y; prm.states[3 * n + 2] = th;
      const double* g = prm.fgoal + 3 * n;
      const double gx = dsub(x, g[0]), gy = dsub(y, g[1]);
      const int arr = (prm.arrived[n] != 0 || sqrt(ddot(gx, gy, gx, gy)) < g[2]) ? 1 : 0;
      prm.arrived[n] = arr;
      if (out_arrived) out_arrived[n] = arr;
      double sn, cs;
      sincos(th, &sn, &cs);
#pragma unroll
      for (int v = 0; v < kWorldMaxVertices; ++v) {  // constant indices into the parameter array
        const double px = prm.robot_v[2 * v], py = prm.robot_v[2 * v + 1];
        f_x[k][v] = dadd(x, dsub(dmul(cs, px), dmul(sn, py)));
        f_y[k][v] = dadd(y, dadd(dmul(sn, px), dmul(cs, py)));
      }
      f_v[k][0] = vx; f_v[k][1] = vy;
    }
    for (int o = o0 + (int)threadIdx.x; o < o1; o += blockDim.x) {
      double cx, cy;
      world_move_obstacle(prm, env, o, cx, cy);
    }
    __syncthreads();  // bodies, velocities and the moved obstacle rows are visible to the whole CTA
    for (int w = threadIdx.x >> 5; w < K; w += nw) {  // warp-uniform
      const size_t n = (size_t)b * K + w;
      double best = INFINITY;
      for (int o = o0 + lane; o < o1; o += 32) {
        const double* row = prm.obs + (size_t)kWorldObsCols * o;
        const double c = world_obstacle_clearance(prm, o, row[0], row[1], f_x[w], f_y[w], nr);
        best = fmin(best, c > 0.0 ? c : 0.0);
      }
      if (lane < K && lane != w) {
        const double c = world_robot_clearance(WorldRobot{f_x[w], f_y[w], nr}, WorldRobot{f_x[lane], f_y[lane], nr});
        best = fmin(best, c > 0.0 ? c : 0.0);
      }
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) best = fmin(best, __shfl_xor_sync(0xffffffffu, best, m));
      if (lane == 0) {
        const int col = (prm.collided[n] != 0 || best <= 0.0) ? 1 : 0;
        prm.collided[n] = col;
        prm.fvel[2 * n] = col ? 0.0 : f_v[w][0];
        prm.fvel[2 * n + 1] = col ? 0.0 : f_v[w][1];
        if (out_collided) out_collided[n] = col;
        if (clearance) clearance[n] = (float)best;
      }
    }
  }
}

}  // namespace nb
