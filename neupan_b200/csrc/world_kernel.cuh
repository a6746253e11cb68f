// Batched 2-D world for closed-loop runs of B planners: what IR-SIM does between two planner calls (example/run_exp.py:27-56,
// env.get_lidar_scan / env.step / env.done), for B environments at once and without leaving the device.
//
// Scene: per environment a ragged list of obstacles -- circles (centre, radius), convex polygons (3..8 vertices) and outlines (any
// simple polygon of 3..16 vertices, convex or not; kind 1), vertices stored relative to the centre so that motion only moves the
// centre -- each with a constant world-frame velocity, an axis-aligned rectangle in which moving obstacles bounce, the robot (the
// planner's robot polygon) and its goal.
//
//   world_scan_kernel   one CTA per environment (grid-stride): the environment's circles and polygon edges (convex and outline
//                       alike) are staged in shared memory in world coordinates, then one thread per beam finds the first boundary
//                       crossing with t > 0
//   world_step_kernel   one warp per environment: obstacles move (reflecting at the rectangle), the robot integrates its action
//                       unless it has collided, then the exact clearance robot polygon <-> every obstacle, reduced over the warp
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
};

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ddot(double ax, double ay, double bx, double by) { return dadd(dmul(ax, bx), dmul(ay, by)); }
__device__ __forceinline__ double dcross(double ax, double ay, double bx, double by) { return dsub(dmul(ax, by), dmul(ay, bx)); }

// ---- lidar ----------------------------------------------------------------------------------------------------------------

// Beam i leaves the sensor at world angle (theta + off_th) + a_i, a_i = linspace(angle_min, angle_max, R)[i] -- the convention
// nb_scan_to_points inverts.  Its direction is evaluated as the rotation of (cos a_i, sin a_i) by the sensor heading: no
// trigonometry per beam (and none of the argument-reduction slow path, whose call would spill the beam loop's registers).  range = the smallest t > 0 at which the ray crosses an obstacle boundary (a sensor inside an obstacle sees the exit
// crossing); t >= range_max or no crossing is a miss: range_max, velocity 0, hit -1.  Equal t: the lower obstacle index wins, so the
// result does not depend on the order of the tests.
__global__ void __launch_bounds__(256) world_scan_kernel(const WorldParams prm, int max_circ, int max_edges, float* __restrict__ ranges,
                                                         float* __restrict__ velocity, int32_t* __restrict__ hit) {
  extern __shared__ double wsm[];
  double* c_x = wsm;
  double* c_y = c_x + max_circ;
  double* c_r = c_y + max_circ;
  double* e_ax = c_r + max_circ;
  double* e_ay = e_ax + max_edges;
  double* e_bx = e_ay + max_edges;
  double* e_by = e_bx + max_edges;
  int32_t* c_id = reinterpret_cast<int32_t*>(e_by + max_edges);
  int32_t* e_id = c_id + max_circ;
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
    __syncthreads();
    const double x = prm.states[3 * b], y = prm.states[3 * b + 1], th = prm.states[3 * b + 2];
    double sn, cs;
    sincos(th, &sn, &cs);
    const double sx = dadd(x, dsub(dmul(cs, prm.off_x), dmul(sn, prm.off_y)));  // sensor position: robot pose applied to scan_offset
    const double sy = dadd(y, dadd(dmul(sn, prm.off_x), dmul(cs, prm.off_y)));
    double hs, hc;
    sincos(dadd(th, prm.off_th), &hs, &hc);
    for (int i = threadIdx.x; i < R; i += blockDim.x) {
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
      if (!(best < prm.range_max)) { best = prm.range_max; bid = -1; }
      const size_t q = (size_t)b * R + i;
      ranges[q] = (float)best;
      if (velocity) {
        const double* row = prm.obs + (size_t)kWorldObsCols * (o0 + (bid < 0 ? 0 : bid));
        velocity[(size_t)b * 2 * R + i] = bid < 0 ? 0.f : (float)row[2];
        velocity[(size_t)b * 2 * R + R + i] = bid < 0 ? 0.f : (float)row[3];
      }
      if (hit) hit[q] = bid;
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
  const double *x, *y;
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

// ---- step -----------------------------------------------------------------------------------------------------------------

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
    const double a0 = (double)action[2 * b], a1 = (double)action[2 * b + 1];
    double dxs, dys, dth;
    if (prm.kinematics == 2) {  // omni: the (vx, vy) PlannerBatch returns
      dxs = a0; dys = a1; dth = 0.0;
    } else {
      double sn, cs;
      sincos(th, &sn, &cs);
      dxs = dmul(a0, cs); dys = dmul(a0, sn);
      dth = prm.kinematics == 1 ? dmul(a0, tan(a1)) / prm.L : a1;  // acker: v tan(phi) / L; diff: omega
    }
    x = dadd(x, dmul(dxs, prm.dt)); y = dadd(y, dmul(dys, prm.dt)); th = dadd(th, dmul(dth, prm.dt));
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
    double* row = prm.obs + (size_t)kWorldObsCols * o;
    double cx = row[0], cy = row[1], vx = row[2], vy = row[3];
    cx = dadd(cx, dmul(vx, prm.dt));
    cy = dadd(cy, dmul(vy, prm.dt));
    if (vx != 0.0) {  // a moving centre that left the rectangle is mirrored back and its velocity component reversed
      if (cx < env[0]) { cx = dsub(dmul(2.0, env[0]), cx); vx = -vx; }
      else if (cx > env[2]) { cx = dsub(dmul(2.0, env[2]), cx); vx = -vx; }
    }
    if (vy != 0.0) {
      if (cy < env[1]) { cy = dsub(dmul(2.0, env[1]), cy); vy = -vy; }
      else if (cy > env[3]) { cy = dsub(dmul(2.0, env[3]), cy); vy = -vy; }
    }
    row[0] = cx; row[1] = cy; row[2] = vx; row[3] = vy;
    const int v0 = prm.vert_begin[o], nv = prm.vert_begin[o + 1] - v0;
    double c;
    if (nv == 0) {  // circle: distance from the centre to the robot polygon - r
      bool pos = false, neg = false;
      double d = INFINITY;
      for (int k = 0; k < nr; ++k) {
        const int k1 = k + 1 < nr ? k + 1 : 0;
        const double cr = dcross(dsub(rx[k1], rx[k]), dsub(ry[k1], ry[k]), dsub(cx, rx[k]), dsub(cy, ry[k]));
        pos |= cr > 0.0; neg |= cr < 0.0;
        d = fmin(d, world_seg_dist(cx, cy, rx[k], ry[k], rx[k1], ry[k1]));
      }
      c = (pos && neg) ? dsub(d, row[4]) : 0.0;  // centre inside the robot: overlap
    } else if (prm.kind[o] != 0) {
      c = world_outline_clearance(WorldPoly{prm.vertices + 2 * (size_t)v0, cx, cy, nv}, rx, ry, nr);
    } else {        // convex polygon: 0 unless an edge normal separates them, then the smallest vertex-edge distance
      const WorldPoly op{prm.vertices + 2 * (size_t)v0, cx, cy, nv};
      const WorldRobot rp{rx, ry, nr};
      if (world_sat_separates(rp, op) || world_sat_separates(op, rp)) {
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
        c = d;
      } else {
        c = 0.0;
      }
    }
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

}  // namespace nb
