// Obstacle contact in the batched world (nb_world_set_obstacle_contact): the obstacles of an environment whose flag is 1 block each
// other.  This project's reading of IR-SIM, which moves its objects one after another.
//
// Touch: two footprints touch when their clearance is <= 0, as everywhere else in the world, by one predicate per pair of kinds (FP64
// with explicit rounding; every predicate gives the same answer for (i, j) and (j, i), bit for bit):
//   circle - circle     sqrt(dx^2 + dy^2) - (r_i + r_j) <= 0
//   circle - convex     the circle branch of world_obstacle_clearance with the polygon in place of the robot: the centre not strictly
//                       outside the polygon, or the smallest centre-edge distance - r <= 0
//   circle - outline    the centre inside by even-odd, or the smallest centre-edge distance <= r
//   convex - convex     world_convex_clearance <= 0
//   convex - outline    world_outline_clearance with the convex side as PC <= 0
//   outline - outline   two edges meet as closed segments (world_segs_meet), or vertex 0 of either outline lies inside the other
//                       (even-odd)
// Broad phase: a pair is tested only when the footprints' axis-aligned boxes, each widened by kWorldContactPad on every side, meet.  A
// footprint's box is its centre plus its centre-relative box (a circle: -r .. r; a polygon: the smallest and largest vertex offset);
// the widening keeps rounding from dropping a touching pair.
//
// Move rule: in an environment with the flag set, the obstacles move in ascending row order.  An obstacle with v != 0 (after the rvo
// kernel) takes (c', v') = world_obstacle_move, then the first of A (c'x, c'y; v'), B (c'x, cy; v'x, -v'y), C (cx, c'y; -v'x, v'y)
// and D (cx, cy; -v') whose footprint touches no other obstacle of its environment -- the earlier rows at their new centres, the later
// rows at their old ones, static obstacles included -- and, where the map blocks obstacles, not the map either.  D is never tested:
// an earlier obstacle was checked clear of this one's old footprint and the later ones have not moved, so D is admissible whenever
// the start was (checked on the host).  A step whose A touches another obstacle is an obstacle bounce; the map's bounce counter and
// `bounced` flag keep their meaning (A touched the map).  Robots do not block obstacles.  Environments whose flag is 0 move their
// obstacles as the step kernel does (world_move_obstacle, or world_move_obstacle_blocked where the maps block obstacles).
//
// Limits: no swept test (a step longer than the thinner footprint can pass through it); no contact with robots; no momentum or
// elastic response; earlier rows move first.
//
//   world_contact_kernel  one warp per environment (kEp: per live slot, moving its scene's rows), kWorldContactWarps warps per CTA.
//                         The warp stages its environment's centres and centre-relative boxes in shared memory (6 doubles per
//                         obstacle, sized by the largest environment), then walks the obstacles in order: for each candidate the lanes
//                         take the other obstacles j = lane, lane + 32, ... and a warp vote combines them; kMap (the handle's maps block
//                         obstacles somewhere): the lanes also run the map test through world_map_any.  Lane 0 writes the row, the
//                         shared centre and the counters.
//   world_step_contact_kernel  world_step_body without the obstacle move (kMove false): the robots integrate and take their
//                         clearances to the obstacles' new rows.
#pragma once
#include "world_kernel.cuh"

namespace nb {

constexpr int kWorldContactWarps = 4;
constexpr double kWorldContactPad = 1e-6;  // m, the broad phase's widening of each box

// Circle (cx, cy, r) <-> convex polygon p: the circle branch of world_obstacle_clearance (the centre not strictly outside p, or the
// smallest centre-edge distance - r <= 0)
template <class PC>
__device__ __forceinline__ bool world_circle_touches_convex(double cx, double cy, double r, const PC& p) {
  bool pos = false, neg = false;
  double d = INFINITY;
  for (int k = 0; k < p.nv; ++k) {
    const int k1 = k + 1 < p.nv ? k + 1 : 0;
    const double ax = p.vx(k), ay = p.vy(k), bx = p.vx(k1), by = p.vy(k1);
    const double cr = dcross(dsub(bx, ax), dsub(by, ay), dsub(cx, ax), dsub(cy, ay));
    pos |= cr > 0.0; neg |= cr < 0.0;
    d = fmin(d, world_seg_dist(cx, cy, ax, ay, bx, by));
  }
  return !(pos && neg) || dsub(d, r) <= 0.0;
}

// Even-odd test of (px, py) against polygon p (world_outline_clearance's test: an edge that straddles the horizontal line through the
// point toggles it when it crosses that line to the point's right)
template <class P>
__device__ __forceinline__ bool world_inside_outline(const P& p, double px, double py) {
  bool in = false;
  for (int k = 0; k < p.nv; ++k) {
    const int k1 = k + 1 < p.nv ? k + 1 : 0;
    const double ax = p.vx(k), ay = p.vy(k), bx = p.vx(k1), by = p.vy(k1);
    if ((ay > py) != (by > py)) {
      const double cr = dcross(dsub(bx, ax), dsub(by, ay), dsub(px, ax), dsub(py, ay));
      if (by > ay ? cr > 0.0 : cr < 0.0) in = !in;
    }
  }
  return in;
}

// Circle (cx, cy, r) <-> outline p: the centre inside by even-odd, or the smallest centre-edge distance <= r
__device__ __forceinline__ bool world_circle_touches_outline(double cx, double cy, double r, const WorldPoly& p) {
  if (world_inside_outline(p, cx, cy)) return true;
  double d = INFINITY;
  for (int k = 0; k < p.nv; ++k) {
    const int k1 = k + 1 < p.nv ? k + 1 : 0;
    d = fmin(d, world_seg_dist(cx, cy, p.vx(k), p.vy(k), p.vx(k1), p.vy(k1)));
  }
  return d <= r;
}

// Outline <-> outline: two edges meet as closed segments, or vertex 0 of either lies inside the other
__device__ __forceinline__ bool world_outlines_touch(const WorldPoly& a, const WorldPoly& b) {
  for (int k = 0; k < a.nv; ++k) {
    const int k1 = k + 1 < a.nv ? k + 1 : 0;
    const double px = a.vx(k), py = a.vy(k), qx = a.vx(k1), qy = a.vy(k1);
    for (int i = 0; i < b.nv; ++i) {
      const int i1 = i + 1 < b.nv ? i + 1 : 0;
      if (world_segs_meet(px, py, qx, qy, b.vx(i), b.vy(i), b.vx(i1), b.vy(i1))) return true;
    }
  }
  return world_inside_outline(b, a.vx(0), a.vy(0)) || world_inside_outline(a, b.vx(0), b.vy(0));
}

// 0 circle, 1 convex polygon, 2 outline
__device__ __forceinline__ int world_shape_rank(const WorldFootprint& f) { return f.nv == 0 ? 0 : (f.kind != 0 ? 2 : 1); }

// Do two obstacle footprints touch (the predicates of the header)?  The pair is put in rank order first, so a mixed pair runs one
// predicate whichever side it comes from.
__device__ __forceinline__ bool world_footprints_touch(const WorldFootprint& f, const WorldFootprint& g) {
  WorldFootprint a = f, b = g;
  if (world_shape_rank(a) > world_shape_rank(b)) { a = g; b = f; }
  const int ra = world_shape_rank(a), rb = world_shape_rank(b);
  if (rb == 0) {
    const double dx = dsub(a.cx, b.cx), dy = dsub(a.cy, b.cy);
    return dsub(__dsqrt_rn(ddot(dx, dy, dx, dy)), dadd(a.r, b.r)) <= 0.0;
  }
  if (ra == 0) return rb == 1 ? world_circle_touches_convex(a.cx, a.cy, a.r, b.poly()) : world_circle_touches_outline(a.cx, a.cy, a.r, b.poly());
  if (rb == 1) return world_convex_clearance(a.poly(), b.poly()) <= 0.0;
  if (ra == 1) return world_outline_clearance(b.poly(), a.poly()) <= 0.0;
  return world_outlines_touch(a.poly(), b.poly());
}

// The obstacle-contact arrays (read by world_contact_kernel only)
struct WorldContactParams {
  const int32_t* flag;  // (B) 1: the environment's obstacles block each other
  int32_t* bounces;     // (O) steps in which the obstacle's move A touched another obstacle
  int max_n;            // the largest environment's obstacle count (the shared staging per warp)
};

// One warp per unit b (an environment, or with kEp a slot); kMap: the handle's maps block obstacles somewhere (bp and mp are read only
// then).  Shared memory: kWorldContactWarps * 6 * max_n doubles.
template <bool kMap, bool kEp>
__global__ void __maxnreg__(128) world_contact_kernel(const WorldParams prm, const WorldMapParams mp, const WorldBlockParams bp,
                                                                                const WorldContactParams cp) {
  extern __shared__ double csm[];
  const int lane = threadIdx.x & 31, n = cp.max_n;
  double* s_cx = csm + (size_t)(threadIdx.x >> 5) * 6 * n;  // this warp's centres and centre-relative boxes
  double* s_cy = s_cx + n;
  double* s_x0 = s_cy + n;
  double* s_y0 = s_x0 + n;
  double* s_x1 = s_y0 + n;
  double* s_y1 = s_x1 + n;
  for (int b = blockIdx.x * kWorldContactWarps + (int)(threadIdx.x >> 5); b < prm.B; b += gridDim.x * kWorldContactWarps) {  // warp-uniform
    if (kEp && prm.live[b] == 0) continue;
    const int e = kEp ? prm.scene_of[b] : b;
    const int o0 = prm.obs_begin[e], no = prm.obs_begin[e + 1] - o0;
    const double* env = prm.env + (size_t)kWorldEnvCols * e;
    if (cp.flag[e] == 0) {  // each obstacle on its own, as the step kernel moves it
      for (int o = o0 + lane; o < o0 + no; o += 32) {
        if constexpr (kMap) {
          world_move_obstacle_blocked(prm, mp, bp, e, o);
        } else {
          double cx, cy;
          world_move_obstacle(prm, env, o, cx, cy);
        }
      }
      continue;
    }
    __syncwarp();  // the previous environment's tests are done with the staging
    for (int i = lane; i < no; i += 32) {
      const double* row = prm.obs + (size_t)kWorldObsCols * (o0 + i);
      const int v0 = prm.vert_begin[o0 + i], nv = prm.vert_begin[o0 + i + 1] - v0;
      double x0, y0, x1, y1;
      if (nv == 0) {
        x0 = y0 = -row[4]; x1 = y1 = row[4];
      } else {
        const double* rel = prm.vertices + 2 * (size_t)v0;
        x0 = x1 = rel[0]; y0 = y1 = rel[1];
        for (int k = 1; k < nv; ++k) {
          x0 = fmin(x0, rel[2 * k]); x1 = fmax(x1, rel[2 * k]);
          y0 = fmin(y0, rel[2 * k + 1]); y1 = fmax(y1, rel[2 * k + 1]);
        }
      }
      s_cx[i] = row[0]; s_cy[i] = row[1];
      s_x0[i] = x0; s_y0[i] = y0; s_x1[i] = x1; s_y1[i] = y1;
    }
    __syncwarp();
    const bool mapb = kMap && bp.block[e] != 0;
    for (int i = 0; i < no; ++i) {  // warp-uniform
      const int o = o0 + i;
      double* row = prm.obs + (size_t)kWorldObsCols * o;
      const double x = row[0], y = row[1];
      const bool moves = row[2] != 0.0 || row[3] != 0.0;
      double cx, cy, vx, vy;
      world_obstacle_move(row, env, prm.dt, cx, cy, vx, vy);
      bool obs_a = false, map_a = false;
      int take = 0;  // 0 A, 1 B, 2 C, 3 D
      if (moves) {
        WorldFootprint f = world_footprint(prm, o, cx, cy);
        for (take = 0; take < 3; ++take) {
          f.cx = take == 2 ? x : cx;
          f.cy = take == 1 ? y : cy;
          const double ax0 = dsub(dadd(f.cx, s_x0[i]), kWorldContactPad), ax1 = dadd(dadd(f.cx, s_x1[i]), kWorldContactPad);
          const double ay0 = dsub(dadd(f.cy, s_y0[i]), kWorldContactPad), ay1 = dadd(dadd(f.cy, s_y1[i]), kWorldContactPad);
          bool hit = false;
          for (int j = lane; j < no && !hit; j += 32) {
            if (j == i) continue;
            const double bx0 = dsub(dadd(s_cx[j], s_x0[j]), kWorldContactPad), bx1 = dadd(dadd(s_cx[j], s_x1[j]), kWorldContactPad);
            const double by0 = dsub(dadd(s_cy[j], s_y0[j]), kWorldContactPad), by1 = dadd(dadd(s_cy[j], s_y1[j]), kWorldContactPad);
            if (ax1 < bx0 || bx1 < ax0 || ay1 < by0 || by1 < ay0) continue;
            hit = world_footprints_touch(f, world_footprint(prm, o0 + j, s_cx[j], s_cy[j]));
          }
          const bool to = __any_sync(0xffffffffu, hit);
          bool tm = false;
          if (mapb && (take == 0 || !to))
            tm = __any_sync(0xffffffffu, world_footprint_touches(mp.maps[mp.env_map[e]], mp.bits, f, lane, 32));
          if (take == 0) { obs_a = to; map_a = tm; }
          if (!to && !tm) break;
        }
      }
      if (lane == 0) {
        if (take == 1) { cy = y; vy = -vy; }
        else if (take == 2) { cx = x; vx = -vx; }
        else if (take == 3) { cx = x; cy = y; vx = -vx; vy = -vy; }
        row[0] = cx; row[1] = cy; row[2] = vx; row[3] = vy;
        s_cx[i] = cx; s_cy[i] = cy;
        if (obs_a) cp.bounces[o] += 1;
        if (mapb) {
          if (map_a) bp.bounces[o] += 1;
          bp.bounced[o] = map_a ? 1 : 0;
        }
      }
      __syncwarp();  // the new centre is visible to every lane before the next obstacle's tests
    }
  }
}

// Obstacle contact: world_step_body without the obstacle move (world_contact_kernel has moved them).  kEp: episode mode.
// __maxnreg__(128) as in world_step_ep_kernel.
template <bool kMap, bool kEp>
__global__ void __maxnreg__(128) world_step_contact_kernel(const WorldParams prm, const WorldMapParams mp, const float* __restrict__ action,
                                                           int32_t* __restrict__ out_collided, int32_t* __restrict__ out_arrived,
                                                           float* __restrict__ clearance) {
  world_step_body<kMap, kEp, false, false>(prm, mp, WorldBlockParams{}, action, out_collided, out_arrived, clearance);
}

}  // namespace nb
