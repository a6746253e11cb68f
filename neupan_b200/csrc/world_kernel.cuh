// Batched 2-D world for closed-loop runs of B planners: what IR-SIM does between two planner calls (example/run_exp.py:27-56,
// env.get_lidar_scan / env.step / env.done), for B environments at once and without leaving the device.
//
// Scene: per environment a ragged list of obstacles -- circles (centre, radius), convex polygons (3..8 vertices) and outlines (any
// simple polygon of 3..16 vertices, convex or not; kind 1), vertices stored relative to the centre so that motion only moves the
// centre -- each with a constant world-frame velocity, an axis-aligned rectangle in which moving obstacles bounce, and K robots
// (1 <= K <= 16: nb_world_set_fleet, or one per environment from the scenes' own start and goal) of the planner's robot polygon,
// each with its goal.  Robot k of environment b is row n = b K + k of every per-robot array, whatever K is.  Mixed fleets
// (nb_world_set_fleet_ex): every robot has a type (rtype, zeros without a mix), a row of the type table (polygon, kinematics,
// wheelbase, circumradius); the kernels read a robot's body and motion model from its type, indexing global memory (a run-time
// index into a kernel parameter array would copy it to local memory).
//
//   world_scan_kernel  one CTA per environment (grid-stride): the environment's circles and polygon edges (convex and outline
//                      alike) and, with K > 1, the K robot bodies (edges tagged with their owner) are staged in shared memory in
//                      world coordinates with each robot's sensor pose, then one thread per beam of the K R beams finds the first
//                      boundary crossing with t > 0; a beam skips its own robot's edges
//   world_step_kernel  one CTA per floor(8 / K) environments (K <= 4) or per environment, at most 8 warps: the robots integrate
//                      (Jacobi: from the states at the start of the step), their world vertices and velocities go to shared memory
//                      and the obstacles move (reflecting at the rectangle); after a barrier one warp per robot takes the exact
//                      clearance to every obstacle of its environment and to every other robot of it (convex-convex, symmetric bit
//                      for bit), then a warp min
//
// Several robots (this project's reading of an IR-SIM world whose robot: section lists several robots): a beam also tests the bodies
// of the other K - 1 robots (the robot polygon at their current state), never its own; a robot hit reports index O_b + j (O_b the
// environment's obstacle count), so at equal t an obstacle wins, and the world-frame velocity of the action that robot integrated in
// the last step (0 before the first step and once it has collided; translation only, omega x r left out).  collided is sticky and
// freezes a robot, which stays in the scene; arrived is sticky and an arrived robot stays in the scene.
//
// Occupancy maps (nb_world_set_maps; this project's reading of IR-SIM's `world: obstacle_map:`): an environment may carry one static
// grid of W x H square cells of side r whose origin (x0, y0) is the lower-left corner of cell (0, 0); cell (i, j) is
// [X(i), X(i+1)] x [Y(j), Y(j+1)] with X(i) = dadd(x0, dmul((double)i, r)), Y(j) likewise -- every corner is computed this way,
// nothing is accumulated.  Cells outside the grid are free (a border is a wall only if the map draws one).  A map is a kind of
// scene, not an obstacle: the obstacle rows do not change, and unless the map blocks obstacles (nb_world_set_map_contact, "obstacles
// in occupancy maps" below) reactive obstacles do not see it and moving obstacles pass over it.
// Both kernels take the map path as a compile-time variant (kMap), launched only when some environment of the handle has a map:
//   scan  after the shape and robot tests, the beam walks the grid cell by cell (world_map_cast) and reports the first t > 0 at
//         which it crosses from a cell of one state into a cell of the other, with index O_b + K (after the obstacles and the
//         robots, so at equal t they win and the walk stops at the current best) and velocity 0.  Every crossing is
//         (boundary - s) / d from the cell index.  The sensor's cell is (floor((s_x - x0) / r), ...) corrected by one step so that
//         X(i) <= s_x < X(i+1): a sensor on a grid line lies in the cell above / to the right of it, and a beam running along that
//         line sees that row (column) only.  At a corner (t_x == t_y) the beam enters the x-neighbour, the y-neighbour and the
//         diagonal cell at once: a crossing if any of the three differs, and the walk continues from the diagonal cell.  A sensor
//         outside the grid enters through its box; a sensor in an occupied cell sees the exit crossing.
//   step  m = min(window, the clearance to the occupied cells that meet the robot's world bounding box grown by window, each
//         cell a 4-vertex CCW polygon through world_convex_clearance), which is the exact clearance to the map whenever it is
//         <= window; the robot's clearance is min(obstacles, robots, m) and m <= 0 sets collided.
// There is no sub-cell geometry.
//
// Obstacle contact (nb_world_set_obstacle_contact; semantics, predicates and limits in world_contact_kernel.cuh): where an
// environment's flag is 1 its obstacles block each other.  They move one at a time in row order, each taking the first of the
// candidates A (the move), B (x only), C (y only), D (stay) whose footprint touches no other obstacle where it stands at that moment
// (nor a map that blocks obstacles), so no moving obstacle ever touches another.  Robots are not blockers.  A handle with a flag set
// moves its obstacles in world_contact_kernel and steps with world_step_body<..., kMove = false>; a handle without one launches the
// kernels above unchanged.
//
// Actuation limits and noise (nb_world_set_actuation, nb_world_set_lidar_noise; this project's reading of IR-SIM's vel_min /
// vel_max / acce and its motion and lidar `noise` switches, not a claim of parity).  Each robot type t has vel_min[2], vel_max[2],
// acce[2] and alpha[4] (defaults -inf, +inf, +inf, 0), in the action's own convention (diff (v, omega), acker (v, steering), omni
// (vx, vy)); each robot row n has cmd_prev[2], its last limited command (0 after nb_world_set_scenes / _fleet / _episodes and when a
// slot takes a new scene).  In a step, robot n of type t with action a (converted to double), per component j:
//   lo_j = max(vel_min_j, cmd_prev_j - acce_j dt)   hi_j = min(vel_max_j, cmd_prev_j + acce_j dt)   c_j = min(max(a_j, lo_j), hi_j)
//   cmd_prev <- c;  s0 = sqrt(alpha0 c0^2 + alpha1 c1^2), s1 = sqrt(alpha2 c0^2 + alpha3 c1^2);  u = (c0 + s0 z0, c1 + s1 z1)
// and the robot integrates u (world_integrate); the velocity the scan reports for it is that of u.  The noise is added after the
// limits and not clipped again (IR-SIM's order); a type whose alpha are all 0 draws nothing (u = c).  A collided robot stays frozen
// and its cmd_prev becomes 0.  Reactive obstacles still see the action as given.  Lidar: a beam that hits something (hit >= 0)
// reports clamp(t + range_std z, range_min, range_max), in FP64 before the float cast; a miss, the hit index and the velocity are
// unchanged.  z is a standard normal draw from the counter-based streams below, keyed by (seed, tag, e, k, n, j): e the environment
// (the scene in episode mode), k the robot within it, n the steps that scene has taken (the host's count in a plain world, the
// slot's episode step t in episode mode; the first scan and step use n = 0), j the component (0, 1) or the beam.  So a run is
// reproducible from its seeds, environment e's noise does not depend on B, two scans without a step between them are equal, and an
// episode is bitwise the plain run of its scene.  Both are compile-time variants (kAct of world_step_body, kNoise of
// world_scan_kernel) launched only when the handle has actuation set or range_std > 0.
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
constexpr int kWorldEnvCols = 10;        // env row: xmin, ymin, xmax, ymax, start x, y, theta, goal x, y, goal threshold (the
                                         // kernels read the rectangle; the host takes the robot's start and goal from the rest)
constexpr int kWorldMaxFleet = 16;       // robots per environment
constexpr int kWorldMaxRobotTypes = 4;   // kinds of robot per handle (type 0 and at most 3 more)
constexpr int kWorldStepMaxWarps = 8;    // world_step_kernel: at most 8 warps per CTA, warp w takes robots w, w + 8

// world_step_kernel's environments per CTA: floor(8 / K) up to K = 4 (a CTA of at most 8 warps, one per robot), else 1
__host__ __device__ constexpr int world_step_envs(int K) { return K <= 4 ? kWorldStepMaxWarps / K : 1; }

// One kind of robot (nb_world_robot_type; type 0 is the robot of nb_world_config): a row of the handle's device type table.
struct WorldRobotType {
  double v[2 * kWorldMaxVertices];  // polygon in its own frame: x0, y0, x1, y1, ... (zero past nv)
  double L;                         // wheelbase (acker)
  double r;                         // circumradius about the state point (a reactive obstacle's neighbour circle)
  int32_t kinematics, nv;           // NB_KIN_*, 3..8 vertices
};

struct WorldParams {
  int B, R;
  double dt, range_max;
  double off_x, off_y, off_th;
  const WorldRobotType* types;            // (T + 1) the type table
  const int32_t* rtype;                   // (B K) each robot's type (all 0 without a mix)
  const double* beam_cs;                  // (R, 2) cos, sin of a_i = linspace(angle_min, angle_max, R)[i] (libm, on the host)
  const int32_t* obs_begin;               // (B + 1) offsets into the obstacle rows
  const int32_t* vert_begin;              // (O + 1) offsets into vertices; an empty range is a circle
  const int32_t* slot;                    // (O) circle: rank among the env's circles; polygon: index of its first edge in the env
  const int32_t* counts;                  // (B, 2) circles, polygon edges of the environment
  const int32_t* kind;                    // (O) 0: circle or convex polygon, 1: outline
  const double* vertices;                 // (V, 2) relative to the obstacle's centre
  const double* env;                      // (B, kWorldEnvCols)
  double* obs;                            // (O, kWorldObsCols) -- centres and velocities change
  int K;                                  // robots per environment
  double* states;                         // (B K, 3) x, y, theta
  int32_t* collided;                      // (B K) sticky
  int32_t* arrived;                       // (B K) sticky
  const double* fgoal;                    // (B K, 3) goal x, y, threshold of every robot
  double* fvel;                           // (B K, 2) world-frame velocity of each robot's last step
  // episode mode (nb_world_set_episodes; read by the kEp instantiations only): B is then the slot count, slot b runs scene
  // scene_of[b] while live[b] != 0; every per-scene array above is indexed by the scene, every per-call input and output by the slot
  const int32_t* scene_of;                // (slots)
  const int32_t* live;                    // (slots) 0: idle, its scene frozen
  float* ep_clear;                        // (slots K) this step's clearance of each slot robot, for world_advance_kernel
};

constexpr int kWorldMaxMapSide = 8192;  // cells per side of an occupancy map

// One occupancy map (nb_world_map) as the kernels read it: rows of `words` = ceil(W / 32) uint32 words from bits + off, row j
// being y index j, bit (i mod 32) of word i / 32 being cell (i, j).
struct WorldMap {
  double x0, y0, r;
  int64_t off;
  int32_t W, H, words, pad_;
};

struct WorldMapParams {
  const WorldMap* maps;     // (P)
  const uint32_t* bits;     // every map's words back to back
  const int32_t* env_map;   // (B) the environment's map, -1 for none
  double window;            // the step's search distance (0, 10] m
};

constexpr int kWorldActCols = 10;  // actuation row of a robot type: vel_min[2], vel_max[2], acce[2], alpha[4]

// Actuation limits, motion noise and lidar noise (read by the kAct / kNoise instantiations only)
struct WorldNoiseParams {
  const double* act;    // (kWorldMaxRobotTypes, kWorldActCols) per robot type (step)
  double* cmd;          // (B K, 2) cmd_prev of every robot row (step)
  const int32_t* ep_t;  // (slots) the steps of each slot's current episode (episode mode)
  uint64_t n;           // plain world: the steps taken since the robots were placed
  uint64_t seed;        // the motion seed (step) or the lidar seed (scan)
  double range_min, range_std;  // scan
};

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ddot(double ax, double ay, double bx, double by) { return dadd(dmul(ax, bx), dmul(ay, by)); }
__device__ __forceinline__ double dcross(double ax, double ay, double bx, double by) { return dsub(dmul(ax, by), dmul(ay, bx)); }

// ---- counter-based random streams ------------------------------------------------------------------------------------------

constexpr uint64_t kSplitMixGamma = 0x9E3779B97F4A7C15ull;
// domain tags of the noise streams, so that they are independent of each other and of the reactive obstacles' goal draws
constexpr uint64_t kNoiseTagMotion = 0x6D6F74696F6E0001ull;
constexpr uint64_t kNoiseTagLidar = 0x6C69646172000002ull;

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

// The noise stream of robot k of environment e at step n under a domain tag: the robot's goal-draw style key with the tag mixed in,
// then output n of it as the seed of the step's draws
__host__ __device__ __forceinline__ uint64_t world_noise_key(uint64_t seed, uint64_t tag, int e, int k, uint64_t n) {
  return splitmix64_at(splitmix64_mix(world_rvo_key(seed, e, k) ^ tag), n);
}

// Draw j of a step's stream: Box-Muller from outputs 2j and 2j + 1, z = sqrt(-2 log(1 - u1)) cos(2 pi u2) (1 - u1 >= 2^-53, so
// z is finite).  Only log and cos are not correctly rounded.
__device__ __forceinline__ double world_normal(uint64_t key, int j) {
  const double u1 = world_u01(splitmix64_at(key, 2 * (uint64_t)j)), u2 = world_u01(splitmix64_at(key, 2 * (uint64_t)j + 1));
  return dmul(sqrt(dmul(-2.0, log(dsub(1.0, u1)))), cos(dmul(6.283185307179586, u2)));
}

// ---- occupancy maps ---------------------------------------------------------------------------------------------------------

// grid line k of an axis: lo + k r (X(k) or Y(k))
__device__ __forceinline__ double world_map_line(double lo, double r, int k) { return dadd(lo, dmul((double)k, r)); }

// floor((s - lo) / r) clamped to -1..n (every index past either end is a free cell alike)
__device__ __forceinline__ int world_map_floor(double s, double lo, double r, int n) {
  const double f = floor(dsub(s, lo) / r);
  return f < -1.0 ? -1 : (f > (double)n ? n : (int)f);
}

__device__ __forceinline__ bool world_map_occupied(const WorldMap& m, const uint32_t* bits, int i, int j) {
  if (i < 0 || i >= m.W || j < 0 || j >= m.H) return false;
  return (__ldg(bits + m.off + (int64_t)j * m.words + (i >> 5)) >> (i & 31)) & 1u;
}

// The cell of coordinate s on an axis of n cells: world_map_floor, corrected by one step so that line(i) <= s < line(i + 1)
__device__ __forceinline__ int world_map_cell(double s, double lo, double r, int n) {
  int i = world_map_floor(s, lo, r, n);
  if (i > -1 && s < world_map_line(lo, r, i)) --i;
  else if (i < n && s >= world_map_line(lo, r, i + 1)) ++i;
  return i;
}

// The next grid line that a ray from s along d (in cell i of n) crosses on this axis: t = (line(k) - s) / d, and ni the cell past
// it (an index before the grid jumps to its first line); INFINITY when d == 0
__device__ __forceinline__ double world_map_next(double s, double d, double lo, double r, int i, int n, int& ni) {
  int k;
  if (d > 0.0) { k = i < 0 ? 0 : i + 1; ni = k; }
  else if (d < 0.0) { k = i >= n ? n : i; ni = k - 1; }
  else return INFINITY;
  return dsub(world_map_line(lo, r, k), s) / d;
}

// The first t in (0, lim) at which the ray s + t d crosses from a cell of one state into a cell of the other (the corner rule of
// the header), INFINITY when there is none before lim.  Each t comes from the cell index, none is accumulated.
__device__ __forceinline__ double world_map_cast(const WorldMap& m, const uint32_t* bits, double sx, double sy, double dx, double dy,
                                                 double lim) {
  int i = world_map_cell(sx, m.x0, m.r, m.W), j = world_map_cell(sy, m.y0, m.r, m.H), ni = i, nj = j;
  bool cur = world_map_occupied(m, bits, i, j);
  double tx = world_map_next(sx, dx, m.x0, m.r, i, m.W, ni), ty = world_map_next(sy, dy, m.y0, m.r, j, m.H, nj);
  while (true) {
    // outside the grid on an axis and not heading into it: every cell left is free
    if ((i < 0 && !(dx > 0.0)) || (i >= m.W && !(dx < 0.0)) || (j < 0 && !(dy > 0.0)) || (j >= m.H && !(dy < 0.0))) break;
    const double t = fmin(tx, ty);
    if (!(t < lim)) break;
    bool changed;
    if (tx < ty) {
      const bool s = world_map_occupied(m, bits, ni, j);
      changed = s != cur; cur = s; i = ni;
      tx = world_map_next(sx, dx, m.x0, m.r, i, m.W, ni);
    } else if (ty < tx) {
      const bool s = world_map_occupied(m, bits, i, nj);
      changed = s != cur; cur = s; j = nj;
      ty = world_map_next(sy, dy, m.y0, m.r, j, m.H, nj);
    } else {  // a corner: the x-neighbour, the y-neighbour and the diagonal cell at once
      const bool a = world_map_occupied(m, bits, ni, j), c = world_map_occupied(m, bits, i, nj), s = world_map_occupied(m, bits, ni, nj);
      changed = a != cur || c != cur || s != cur; cur = s; i = ni; j = nj;
      tx = world_map_next(sx, dx, m.x0, m.r, i, m.W, ni);
      ty = world_map_next(sy, dy, m.y0, m.r, j, m.H, nj);
    }
    if (changed && t > 0.0) return t;
  }
  return INFINITY;
}

// ---- lidar ----------------------------------------------------------------------------------------------------------------

// Beam i of robot k leaves that robot's sensor at world angle (theta + off_th) + a_i, a_i = linspace(angle_min, angle_max, R)[i] --
// the convention nb_scan_to_points inverts.  Its direction is evaluated as the rotation of (cos a_i, sin a_i) by the sensor heading:
// no trigonometry per beam (and none of the argument-reduction slow path, whose call would spill the beam loop's registers); the
// sensor poses are computed once per environment and staged in shared memory.  range = the smallest t > 0 at which the ray crosses an
// obstacle boundary or, with K > 1, the body of another robot of the environment (a sensor inside an obstacle or another robot sees
// the exit crossing); t >= range_max or no crossing is a miss: range_max, velocity 0, hit -1.  Equal t: the lower index wins
// (obstacles 0..O_b - 1, then robot j as O_b + j), so the result does not depend on the order of the tests.
// max_redges: the largest environment's robot edge count (the sum of its robots' vertex counts with K > 1, else 0); robot k's edges
// follow those of robots 0 .. k - 1, each robot's polygon that of its own type.  kMap: then the environment's map (world_map_cast,
// index O_b + K, velocity 0); mp is not read without it.  kEp (episode mode): the CTA's unit b is a slot, which scans the robots of
// scene scene_of[b] (an idle slot its frozen scene) into slot rows b K + k.  kNoise (range_std > 0): a hit's range gets the lidar
// noise of the header, draw i of robot k's lidar stream at the scene's step n; nz is not read without it.
template <bool kMap, bool kEp, bool kNoise = false>
__global__ void __launch_bounds__(256) world_scan_kernel(const WorldParams prm, const WorldMapParams mp, int max_circ, int max_edges, int max_redges,
                                                         float* __restrict__ ranges, float* __restrict__ velocity, int32_t* __restrict__ hit,
                                                         const WorldNoiseParams nz) {
  extern __shared__ double wsm[];
  __shared__ double s_sx[kWorldMaxFleet], s_sy[kWorldMaxFleet], s_hc[kWorldMaxFleet], s_hs[kWorldMaxFleet];  // sensor poses
  __shared__ int s_nre;  // the environment's robot edges
  const int K = prm.K;
  const int mre = K > 1 ? max_redges : 0;  // a single robot stages no robot edges
  double* r_ax = wsm;
  double* r_ay = r_ax + mre;
  double* r_bx = r_ay + mre;
  double* r_by = r_bx + mre;
  double* c_x = r_by + mre;
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
    const int e = kEp ? prm.scene_of[b] : b;  // the scene: obstacle and robot rows; b: the output rows
    const int o0 = prm.obs_begin[e], o1 = prm.obs_begin[e + 1];
    const int nc = prm.counts[2 * e], ne = prm.counts[2 * e + 1];
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
      const size_t n = (size_t)e * K + k;
      const double x = prm.states[3 * n], y = prm.states[3 * n + 1], th = prm.states[3 * n + 2];
      double sn, cs;
      sincos(th, &sn, &cs);
      s_sx[k] = dadd(x, dsub(dmul(cs, prm.off_x), dmul(sn, prm.off_y)));  // sensor position: robot pose applied to scan_offset
      s_sy[k] = dadd(y, dadd(dmul(sn, prm.off_x), dmul(cs, prm.off_y)));
      double hs, hc;
      sincos(dadd(th, prm.off_th), &hs, &hc);
      s_hc[k] = hc; s_hs[k] = hs;
      if (K > 1) {
        int e0 = 0;  // robot k's first edge: after the edges of robots 0 .. k - 1
        for (int j = 0; j < k; ++j) e0 += prm.types[prm.rtype[(size_t)e * K + j]].nv;
        const WorldRobotType* ty = prm.types + prm.rtype[n];
        const int nr = ty->nv;
        if (k == K - 1) s_nre = e0 + nr;
        // world vertex v (the step kernel's arithmetic) starts edge v and ends edge v - 1: one pass, no vertex arrays in registers
#pragma unroll 1
        for (int v = 0; v < nr; ++v) {
          const double px = ty->v[2 * v], py = ty->v[2 * v + 1];
          const double wx = dadd(x, dsub(dmul(cs, px), dmul(sn, py))), wy = dadd(y, dadd(dmul(sn, px), dmul(cs, py)));
          const int e = e0 + v, ep = e0 + (v == 0 ? nr - 1 : v - 1);
          r_ax[e] = wx; r_ay[e] = wy; r_id[e] = k;
          r_bx[ep] = wx; r_by[ep] = wy;
        }
      }
    }
    __syncthreads();
    const int nobs = o1 - o0, nre = K > 1 ? s_nre : 0;
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
      if constexpr (kMap) {  // the highest index: only a strictly closer crossing counts, so the walk stops at best
        const int mi = mp.env_map[e];
        if (mi >= 0) {
          const double t = world_map_cast(mp.maps[mi], mp.bits, sx, sy, dx, dy, fmin(best, prm.range_max));
          if (t < best) { best = t; bid = nobs + K; }
        }
      }
      if (!(best < prm.range_max)) { best = prm.range_max; bid = -1; }
      if constexpr (kNoise) {
        if (bid >= 0) {
          const uint64_t step = kEp ? (uint64_t)nz.ep_t[b] : nz.n;
          const double r = dadd(best, dmul(nz.range_std, world_normal(world_noise_key(nz.seed, kNoiseTagLidar, e, k, step), i)));
          best = fmin(fmax(r, nz.range_min), prm.range_max);
        }
      }
      const size_t n = (size_t)b * K + k;
      ranges[n * R + i] = (float)best;
      if (velocity) {
        float vx = 0.f, vy = 0.f;
        if (kMap && bid == nobs + K) {
          // the map does not move
        } else if (bid >= nobs) {
          const double* fv = prm.fvel + 2 * ((size_t)e * K + (bid - nobs));
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
// The convex side is any vertex accessor (vx, vy, nv): the robot's world vertices, or an occupancy cell (WorldCell) when an outline
// obstacle meets a map.
template <class PC>
__device__ __forceinline__ double world_outline_clearance(const WorldPoly& op, const PC& c) {
  const int nr = c.nv;
  bool in = false;
  for (int k = 0; k < op.nv; ++k) {
    const int k1 = k + 1 < op.nv ? k + 1 : 0;
    const double ax = op.vx(k), ay = op.vy(k), bx = op.vx(k1), by = op.vy(k1);
    for (int i = 0; i < nr; ++i) {
      const int i1 = i + 1 < nr ? i + 1 : 0;
      if (world_segs_meet(c.vx(i), c.vy(i), c.vx(i1), c.vy(i1), ax, ay, bx, by)) return 0.0;
    }
    if ((ay > c.vy(0)) != (by > c.vy(0))) {
      const double cr = dcross(dsub(bx, ax), dsub(by, ay), dsub(c.vx(0), ax), dsub(c.vy(0), ay));
      if (by > ay ? cr > 0.0 : cr < 0.0) in = !in;
    }
  }
  if (in) return 0.0;
  {
    const double px = op.vx(0), py = op.vy(0);
    bool pos = false, neg = false;
    for (int k = 0; k < nr; ++k) {
      const int k1 = k + 1 < nr ? k + 1 : 0;
      const double cr = dcross(dsub(c.vx(k1), c.vx(k)), dsub(c.vy(k1), c.vy(k)), dsub(px, c.vx(k)), dsub(py, c.vy(k)));
      pos |= cr > 0.0; neg |= cr < 0.0;
    }
    if (!(pos && neg)) return 0.0;
  }
  double d = INFINITY;
  for (int k = 0; k < op.nv; ++k) {
    const int k1 = k + 1 < op.nv ? k + 1 : 0;
    const double ax = op.vx(k), ay = op.vy(k), bx = op.vx(k1), by = op.vy(k1);
    for (int i = 0; i < nr; ++i) d = fmin(d, world_seg_dist(c.vx(i), c.vy(i), ax, ay, bx, by));
  }
  for (int k = 0; k < nr; ++k) {
    const int k1 = k + 1 < nr ? k + 1 : 0;
    for (int i = 0; i < op.nv; ++i) d = fmin(d, world_seg_dist(op.vx(i), op.vy(i), c.vx(k), c.vy(k), c.vx(k1), c.vy(k1)));
  }
  return d;
}

// ---- step ----------------------------------------------------------------------------------------------------------------

// World-frame translation rate of a robot's action at heading th: diff / acker v (cos th, sin th), omni the (vx, vy) PlannerBatch
// returns.
__device__ __forceinline__ void world_robot_velocity(int kinematics, double a0, double a1, double th, double& vx, double& vy) {
  if (kinematics == 2) {
    vx = a0; vy = a1;
  } else {
    double sn, cs;
    sincos(th, &sn, &cs);
    vx = dmul(a0, cs); vy = dmul(a0, sn);
  }
}

// One step of the motion models from (x, y, th); (vx, vy) is the world-frame translation rate it used (world_robot_velocity, with
// the heading before the step), for a robot of the given kinematics and wheelbase L.
__device__ __forceinline__ void world_integrate(int kinematics, double L, double dt, double a0, double a1, double& x, double& y, double& th,
                                                double& vx, double& vy) {
  world_robot_velocity(kinematics, a0, a1, th, vx, vy);
  // omni: no turn; acker: v tan(phi) / L; diff: omega
  const double dth = kinematics == 2 ? 0.0 : (kinematics == 1 ? dmul(a0, tan(a1)) / L : a1);
  x = dadd(x, dmul(vx, dt)); y = dadd(y, dmul(vy, dt)); th = dadd(th, dmul(dth, dt));
}

// The actuation stage of the header for robot row n (robot k of scene e) of type t at the scene's step n_step: the action (a0, a1)
// becomes the limited command c, written to cmd_prev, plus the motion noise (none when the type's alpha are all 0).
__device__ __forceinline__ void world_actuate(const WorldNoiseParams& nz, double dt, int t, size_t n, int e, int k, uint64_t n_step, double& a0,
                                              double& a1) {
  const double* A = nz.act + (size_t)kWorldActCols * t;
  double* cmd = nz.cmd + 2 * n;
  double c[2] = {a0, a1};
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const double r = dmul(A[4 + j], dt);
    const double lo = fmax(A[j], dsub(cmd[j], r)), hi = fmin(A[2 + j], dadd(cmd[j], r));
    c[j] = fmin(fmax(c[j], lo), hi);
    cmd[j] = c[j];
  }
  a0 = c[0]; a1 = c[1];
  if (A[6] != 0.0 || A[7] != 0.0 || A[8] != 0.0 || A[9] != 0.0) {
    const double q0 = dmul(c[0], c[0]), q1 = dmul(c[1], c[1]);
    const double s0 = sqrt(dadd(dmul(A[6], q0), dmul(A[7], q1))), s1 = sqrt(dadd(dmul(A[8], q0), dmul(A[9], q1)));
    const uint64_t key = world_noise_key(nz.seed, kNoiseTagMotion, e, k, n_step);
    a0 = dadd(c[0], dmul(s0, world_normal(key, 0)));
    a1 = dadd(c[1], dmul(s1, world_normal(key, 1)));
  }
}

// The move of an obstacle row by v dt; a moving centre that left the rectangle env is mirrored back and its velocity component
// reversed: the new centre (cx, cy) and velocity (vx, vy).
__device__ __forceinline__ void world_obstacle_move(const double* row, const double* env, double dt, double& cx, double& cy, double& vx,
                                                    double& vy) {
  vx = row[2]; vy = row[3];
  cx = dadd(row[0], dmul(vx, dt));
  cy = dadd(row[1], dmul(vy, dt));
  if (vx != 0.0) {
    if (cx < env[0]) { cx = dsub(dmul(2.0, env[0]), cx); vx = -vx; }
    else if (cx > env[2]) { cx = dsub(dmul(2.0, env[2]), cx); vx = -vx; }
  }
  if (vy != 0.0) {
    if (cy < env[1]) { cy = dsub(dmul(2.0, env[1]), cy); vy = -vy; }
    else if (cy > env[3]) { cy = dsub(dmul(2.0, env[3]), cy); vy = -vy; }
  }
}

// Obstacle o moves by world_obstacle_move.  Writes the row and returns the new centre.
__device__ __forceinline__ void world_move_obstacle(const WorldParams& prm, const double* env, int o, double& cx, double& cy) {
  double* row = prm.obs + (size_t)kWorldObsCols * o;
  double vx, vy;
  world_obstacle_move(row, env, prm.dt, cx, cy, vx, vy);
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
  if (prm.kind[o] != 0) return world_outline_clearance(WorldPoly{prm.vertices + 2 * (size_t)v0, cx, cy, nv}, WorldRobot{rx, ry, nr});
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

// Convex <-> convex: 0 unless an edge normal of either separates them (both SAT orders), else the smallest vertex-edge distance both
// ways.  Swapping a and b evaluates the same tests and distances and reduces them with fmin, so the result is symmetric bit for
// bit: two robots that touch collide in the same step.
template <class PA, class PB>
__device__ __forceinline__ double world_convex_clearance(const PA& a, const PB& b) {
  if (!(world_sat_separates(a, b) || world_sat_separates(b, a))) return 0.0;
  double d = INFINITY;
  for (int k = 0; k < b.nv; ++k) {
    const int k1 = k + 1 < b.nv ? k + 1 : 0;
    for (int i = 0; i < a.nv; ++i) d = fmin(d, world_seg_dist(a.vx(i), a.vy(i), b.vx(k), b.vy(k), b.vx(k1), b.vy(k1)));
  }
  for (int k = 0; k < a.nv; ++k) {
    const int k1 = k + 1 < a.nv ? k + 1 : 0;
    for (int i = 0; i < b.nv; ++i) d = fmin(d, world_seg_dist(b.vx(i), b.vy(i), a.vx(k), a.vy(k), a.vx(k1), a.vy(k1)));
  }
  return d;
}

// Robot <-> robot
__device__ __forceinline__ double world_robot_clearance(const WorldRobot& a, const WorldRobot& b) { return world_convex_clearance(a, b); }

// An occupancy cell [xa, xb] x [ya, yb] as a convex polygon: (xa, ya), (xb, ya), (xb, yb), (xa, yb) (CCW)
struct WorldCell {
  double xa, ya, xb, yb;
  static constexpr int nv = 4;
  __device__ __forceinline__ double vx(int k) const { return (k == 1 || k == 2) ? xb : xa; }
  __device__ __forceinline__ double vy(int k) const { return k >= 2 ? yb : ya; }
};

// The robot's (world vertices rx, ry) smallest clearance, clamped at 0, to the occupied cells of map m that meet its bounding box
// grown by window (widened by one cell on each side, so that rounding cannot drop a cell within window); lane `lane` of the warp
// takes the (row, word) pairs lane, lane + 32, ... of that range, skips zero words and visits the set bits.  INFINITY for none.
__device__ __forceinline__ double world_map_clearance(const WorldMap& m, const uint32_t* bits, double window, const double* rx, const double* ry,
                                                      int nr, int lane) {
  double xmin = rx[0], xmax = rx[0], ymin = ry[0], ymax = ry[0];
  for (int k = 1; k < nr; ++k) {
    xmin = fmin(xmin, rx[k]); xmax = fmax(xmax, rx[k]);
    ymin = fmin(ymin, ry[k]); ymax = fmax(ymax, ry[k]);
  }
  const int i0 = max(world_map_floor(dsub(xmin, window), m.x0, m.r, m.W) - 1, 0);
  const int i1 = min(world_map_floor(dadd(xmax, window), m.x0, m.r, m.W) + 1, m.W - 1);
  const int j0 = max(world_map_floor(dsub(ymin, window), m.y0, m.r, m.H) - 1, 0);
  const int j1 = min(world_map_floor(dadd(ymax, window), m.y0, m.r, m.H) + 1, m.H - 1);
  double d = INFINITY;
  if (i0 > i1 || j0 > j1) return d;
  const int w0 = i0 >> 5, nw = (i1 >> 5) - w0 + 1;
  for (int p = lane; p < (j1 - j0 + 1) * nw; p += 32) {
    const int j = j0 + p / nw, wd = w0 + p % nw, lo = i0 - 32 * wd, hi = i1 - 32 * wd;
    uint32_t word = __ldg(bits + m.off + (int64_t)j * m.words + wd);
    if (lo > 0) word &= ~0u << lo;
    if (hi < 31) word &= (2u << hi) - 1u;
    while (word) {
      const int i = 32 * wd + __ffs(word) - 1;
      word &= word - 1u;
      const WorldCell c{world_map_line(m.x0, m.r, i), world_map_line(m.y0, m.r, j), world_map_line(m.x0, m.r, i + 1),
                        world_map_line(m.y0, m.r, j + 1)};
      const double cc = world_convex_clearance(WorldRobot{rx, ry, nr}, c);
      d = fmin(d, cc > 0.0 ? cc : 0.0);
    }
  }
  return d;
}

// ---- obstacles in occupancy maps (nb_world_set_map_contact) -----------------------------------------------------------------
//
// In an environment whose map blocks obstacles, an obstacle touches the map when its footprint has clearance <= 0 to an occupied
// cell (touch counts, as for the robots): a circle when its centre's distance to the closed cell is <= r, a convex polygon by
// world_convex_clearance against the cell, an outline by world_outline_clearance with the cell as the convex side.  Every moving
// obstacle takes the first of these that does not touch the map, (c', v') being the move and mirror of world_move_obstacle from
// (c, v): A (c'x, c'y) with (v'x, v'y); B (c'x, cy) with (v'x, -v'y); C (cx, c'y) with (-v'x, v'y); D (cx, cy) with (-v'x, -v'y).
// D is always taken when A..C touch (the start is clear: checked on the host, then kept by induction).  A step that rejects A is
// a bounce.  Only the occupied cells that meet a bounding box widened by one cell are visited (world_map_any).

// Segment p-q as a two-vertex convex polygon (its two edges are p-q and q-p, whose normals are the segment's normal): SAT and the
// vertex-edge distances of world_convex_clearance then give the segment's distance to a convex polygon (0 when they meet).
struct WorldSeg {
  double px, py, qx, qy;
  static constexpr int nv = 2;
  __device__ __forceinline__ double vx(int k) const { return k ? qx : px; }
  __device__ __forceinline__ double vy(int k) const { return k ? qy : py; }
};

// An obstacle's footprint centred at (cx, cy): a circle of radius r (nv == 0), a convex polygon or an outline (kind 1).
struct WorldFootprint {
  const double* rel;
  double cx, cy, r;
  int nv, kind;
  __device__ __forceinline__ WorldPoly poly() const { return WorldPoly{rel, cx, cy, nv}; }
  // its bounding box (xmin, ymin, xmax, ymax)
  __device__ __forceinline__ void box(double& x0, double& y0, double& x1, double& y1) const {
    if (nv == 0) { x0 = dsub(cx, r); y0 = dsub(cy, r); x1 = dadd(cx, r); y1 = dadd(cy, r); return; }
    x0 = x1 = dadd(cx, rel[0]); y0 = y1 = dadd(cy, rel[1]);
    for (int k = 1; k < nv; ++k) {
      const double x = dadd(cx, rel[2 * k]), y = dadd(cy, rel[2 * k + 1]);
      x0 = fmin(x0, x); x1 = fmax(x1, x); y0 = fmin(y0, y); y1 = fmax(y1, y);
    }
  }
  __device__ __forceinline__ bool touches(const WorldCell& c) const {
    if (nv == 0) {
      if (c.xa <= cx && cx <= c.xb && c.ya <= cy && cy <= c.yb) return true;
      double d = INFINITY;
      for (int k = 0; k < 4; ++k) {
        const int k1 = (k + 1) & 3;
        d = fmin(d, world_seg_dist(cx, cy, c.vx(k), c.vy(k), c.vx(k1), c.vy(k1)));
      }
      return dsub(d, r) <= 0.0;
    }
    return (kind != 0 ? world_outline_clearance(poly(), c) : world_convex_clearance(poly(), c)) <= 0.0;
  }
};

__device__ __forceinline__ WorldFootprint world_footprint(const WorldParams& prm, int o, double cx, double cy) {
  const int v0 = prm.vert_begin[o];
  return WorldFootprint{prm.vertices + 2 * (size_t)v0, cx, cy, prm.obs[(size_t)kWorldObsCols * o + 4], prm.vert_begin[o + 1] - v0, prm.kind[o]};
}

// Is hit(cell) true for an occupied cell of map m that meets [x0, x1] x [y0, y1] widened by one cell on each side?  This thread
// takes the (row, word) pairs first, first + stride, ... of that range (a warp: lane, 32; a thread alone: 0, 1) and stops at its
// first hit; a warp ORs its lanes' answers.
template <class F>
__device__ __forceinline__ bool world_map_any(const WorldMap& m, const uint32_t* bits, double x0, double y0, double x1, double y1, int first,
                                              int stride, const F& hit) {
  const int i0 = max(world_map_floor(x0, m.x0, m.r, m.W) - 1, 0), i1 = min(world_map_floor(x1, m.x0, m.r, m.W) + 1, m.W - 1);
  const int j0 = max(world_map_floor(y0, m.y0, m.r, m.H) - 1, 0), j1 = min(world_map_floor(y1, m.y0, m.r, m.H) + 1, m.H - 1);
  if (i0 > i1 || j0 > j1) return false;
  const int w0 = i0 >> 5, nw = (i1 >> 5) - w0 + 1;
  for (int p = first; p < (j1 - j0 + 1) * nw; p += stride) {
    const int j = j0 + p / nw, wd = w0 + p % nw, lo = i0 - 32 * wd, hi = i1 - 32 * wd;
    uint32_t word = __ldg(bits + m.off + (int64_t)j * m.words + wd);
    if (lo > 0) word &= ~0u << lo;
    if (hi < 31) word &= (2u << hi) - 1u;
    while (word) {
      const int i = 32 * wd + __ffs(word) - 1;
      word &= word - 1u;
      if (hit(WorldCell{world_map_line(m.x0, m.r, i), world_map_line(m.y0, m.r, j), world_map_line(m.x0, m.r, i + 1),
                        world_map_line(m.y0, m.r, j + 1)}))
        return true;
    }
  }
  return false;
}

// Does the footprint touch map m?  One thread (first, stride = 0, 1) or a warp (lane, 32, then __any_sync by the caller).
__device__ __forceinline__ bool world_footprint_touches(const WorldMap& m, const uint32_t* bits, const WorldFootprint& f, int first, int stride) {
  double x0, y0, x1, y1;
  f.box(x0, y0, x1, y1);
  return world_map_any(m, bits, x0, y0, x1, y1, first, stride, [&](const WorldCell& c) { return f.touches(c); });
}

// The map-contact arrays of a handle whose maps block obstacles somewhere (read by the kBlock instantiations only)
struct WorldBlockParams {
  const int32_t* block;  // (B) 1: the environment's map blocks its obstacles
  int32_t* bounces;      // (O) steps in which the obstacle's move A was rejected
  int32_t* bounced;      // (O) 1: rejected in the last step (a reactive obstacle then treats its goal as reached)
};

// world_move_obstacle, then in an environment e whose map blocks obstacles the move rule above for an obstacle that moves (v != 0).
__device__ __forceinline__ void world_move_obstacle_blocked(const WorldParams& prm, const WorldMapParams& mp, const WorldBlockParams& bp, int e, int o) {
  double* row = prm.obs + (size_t)kWorldObsCols * o;
  const double x = row[0], y = row[1];
  const bool moves = row[2] != 0.0 || row[3] != 0.0;
  double cx, cy;
  world_move_obstacle(prm, prm.env + (size_t)kWorldEnvCols * e, o, cx, cy);
  if (bp.block[e] == 0) return;
  int bounced = 0;
  if (moves) {
    const WorldMap& m = mp.maps[mp.env_map[e]];
    WorldFootprint f = world_footprint(prm, o, cx, cy);
    if (world_footprint_touches(m, mp.bits, f, 0, 1)) {
      bounced = 1;
      const double vx = row[2], vy = row[3];
      f.cy = y;
      if (!world_footprint_touches(m, mp.bits, f, 0, 1)) {
        row[1] = y; row[3] = -vy;  // B
      } else {
        f.cx = x; f.cy = cy;
        if (!world_footprint_touches(m, mp.bits, f, 0, 1)) {
          row[0] = x; row[2] = -vx;  // C
        } else {
          row[0] = x; row[1] = y; row[2] = -vx; row[3] = -vy;  // D
        }
      }
      bp.bounces[o] += 1;
    }
  }
  bp.bounced[o] = bounced;
}

// One CTA per E = world_step_envs(K) environments, 32 min(E K, 8) threads (grid = ceil(B / E)); its robots are the slots
// s = n - b0 K of the rows n of its environments b0 .. b0 + E - 1.  Phase 1: thread s integrates robot s from the state at the start
// of the step (unless it has collided), writes its state, arrival flag, world vertices and velocity; every thread moves obstacles.
// Phase 2, after the barrier: one warp per robot (warp w takes slots w, w + 8; a 512-thread CTA would cap the registers at 128 and
// spill) computes its clearance to every obstacle of its environment (lanes over the obstacles: the circle, convex and outline
// branches of world_obstacle_clearance) and to every other robot of it (lane j), a warp min, and lane 0 writes the collision flag,
// the clearance and the velocity the scan reports for the robot (0 once collided).  kMap: the warp also takes min(window, the
// clearance to the environment's map) (world_map_clearance) into the warp min; mp is not read without it.
// kEp (episode mode): the CTA's units are slots b0 .. b0 + E - 1; a live slot steps the robots and obstacles of scene scene_of[b]
// (the scene's rows) and writes its outputs to slot rows q = b K + k, its clearances also to ep_clear; an idle slot's scene is not
// touched, and its outputs are the frozen flags and clearance +inf.
// kMove false (obstacle contact, nb_world_set_obstacle_contact): world_contact_kernel has already moved the obstacles, so phase 1
// integrates the robots only.
// kAct (nb_world_set_actuation): phase 1 limits the action and adds the motion noise first (world_actuate); nz is not read
// without it.
template <bool kMap, bool kEp, bool kBlock, bool kMove = true, bool kAct = false>
__device__ __forceinline__ void world_step_body(const WorldParams& prm, const WorldMapParams& mp, const WorldBlockParams& bp, const float* __restrict__ action,
                                                int32_t* __restrict__ out_collided, int32_t* __restrict__ out_arrived, float* __restrict__ clearance,
                                                const WorldNoiseParams& nz = WorldNoiseParams{}) {
  __shared__ double f_x[kWorldMaxFleet][kWorldMaxVertices], f_y[kWorldMaxFleet][kWorldMaxVertices];  // E K <= 8 or K <= 16 slots
  __shared__ double f_v[kWorldMaxFleet][2];
  __shared__ int f_nv[kWorldMaxFleet];  // each slot's vertex count (its type's)
  const int K = prm.K, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int b0 = blockIdx.x * world_step_envs(K);
  const int nslot = min(world_step_envs(K), prm.B - b0) * K;  // this CTA's robots
  const size_t n0 = (size_t)b0 * K;
  for (int s = threadIdx.x; s < nslot; s += blockDim.x) {
    const size_t q = n0 + s;  // the output row
    const size_t n = kEp ? (size_t)prm.scene_of[b0 + s / K] * K + s % K : q;  // the robot's row
    if (kEp && prm.live[b0 + s / K] == 0) {
      if (out_arrived) out_arrived[q] = prm.arrived[n];
      continue;
    }
    double x = prm.states[3 * n], y = prm.states[3 * n + 1], th = prm.states[3 * n + 2];
    double vx = 0.0, vy = 0.0;
    const WorldRobotType* ty = prm.types + prm.rtype[n];
    if constexpr (kAct) {
      if (prm.collided[n] == 0) {
        double a0 = (double)action[2 * q], a1 = (double)action[2 * q + 1];
        const uint64_t step = kEp ? (uint64_t)nz.ep_t[b0 + s / K] : nz.n;
        world_actuate(nz, prm.dt, prm.rtype[n], n, (int)(n / K), (int)(n % K), step, a0, a1);
        world_integrate(ty->kinematics, ty->L, prm.dt, a0, a1, x, y, th, vx, vy);
      } else {
        nz.cmd[2 * n] = 0.0; nz.cmd[2 * n + 1] = 0.0;
      }
    } else if (prm.collided[n] == 0) {
      world_integrate(ty->kinematics, ty->L, prm.dt, (double)action[2 * q], (double)action[2 * q + 1], x, y, th, vx, vy);
    }
    prm.states[3 * n] = x; prm.states[3 * n + 1] = y; prm.states[3 * n + 2] = th;
    const double* g = prm.fgoal + 3 * n;
    const double gx = dsub(x, g[0]), gy = dsub(y, g[1]);
    const int arr = (prm.arrived[n] != 0 || sqrt(ddot(gx, gy, gx, gy)) < g[2]) ? 1 : 0;
    prm.arrived[n] = arr;
    if (out_arrived) out_arrived[q] = arr;
    double sn, cs;
    sincos(th, &sn, &cs);
#pragma unroll
    for (int v = 0; v < kWorldMaxVertices; ++v) {  // the type's polygon (zero past nv, unused)
      const double px = ty->v[2 * v], py = ty->v[2 * v + 1];
      f_x[s][v] = dadd(x, dsub(dmul(cs, px), dmul(sn, py)));
      f_y[s][v] = dadd(y, dadd(dmul(sn, px), dmul(cs, py)));
    }
    f_v[s][0] = vx; f_v[s][1] = vy;
    f_nv[s] = ty->nv;
  }
  if constexpr (!kMove) {
    // the obstacles have moved
  } else if constexpr (kEp) {  // the slots' scenes are anywhere in the obstacle rows: one live scene after the other
    for (int j = 0; j < nslot / K; ++j) {
      if (prm.live[b0 + j] == 0) continue;
      const int e = prm.scene_of[b0 + j];
      for (int o = prm.obs_begin[e] + (int)threadIdx.x; o < prm.obs_begin[e + 1]; o += blockDim.x) {
        if constexpr (kBlock) {
          world_move_obstacle_blocked(prm, mp, bp, e, o);
        } else {
          double cx, cy;
          world_move_obstacle(prm, prm.env + (size_t)kWorldEnvCols * e, o, cx, cy);
        }
      }
    }
  } else {
    int b = b0;  // the environment of obstacle o: the CTA's obstacle rows are its environments' back to back
    for (int o = prm.obs_begin[b0] + (int)threadIdx.x; o < prm.obs_begin[b0 + nslot / K]; o += blockDim.x) {
      while (o >= prm.obs_begin[b + 1]) ++b;
      if constexpr (kBlock) {
        world_move_obstacle_blocked(prm, mp, bp, b, o);
      } else {
        double cx, cy;
        world_move_obstacle(prm, prm.env + (size_t)kWorldEnvCols * b, o, cx, cy);
      }
    }
  }
  __syncthreads();  // bodies, velocities and the moved obstacle rows are visible to the whole CTA
  for (int s = threadIdx.x >> 5; s < nslot; s += nw) {  // warp-uniform
    const int k = s % K, s0 = s - k;  // robot k of the environment whose robots are the slots s0 .. s0 + K - 1
    const size_t q = n0 + s;          // the output row
    const int b = kEp ? prm.scene_of[b0 + s / K] : b0 + s / K;  // the scene
    const size_t n = kEp ? (size_t)b * K + k : q;                // the robot's row
    if (kEp && prm.live[b0 + s / K] == 0) {
      if (lane == 0) {
        if (out_collided) out_collided[q] = prm.collided[n];
        if (clearance) clearance[q] = INFINITY;
      }
      continue;
    }
    const int nr = f_nv[s];
    double best = INFINITY;
    for (int o = prm.obs_begin[b] + lane; o < prm.obs_begin[b + 1]; o += 32) {
      const double* row = prm.obs + (size_t)kWorldObsCols * o;
      const double c = world_obstacle_clearance(prm, o, row[0], row[1], f_x[s], f_y[s], nr);
      best = fmin(best, c > 0.0 ? c : 0.0);
    }
    if (lane < K && lane != k) {  // each side with its own vertex count: symmetric bit for bit across types too
      const double c = world_robot_clearance(WorldRobot{f_x[s], f_y[s], nr}, WorldRobot{f_x[s0 + lane], f_y[s0 + lane], f_nv[s0 + lane]});
      best = fmin(best, c > 0.0 ? c : 0.0);
    }
    if constexpr (kMap) {
      const int mi = mp.env_map[b];
      if (mi >= 0) best = fmin(best, fmin(mp.window, world_map_clearance(mp.maps[mi], mp.bits, mp.window, f_x[s], f_y[s], nr, lane)));
    }
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) best = fmin(best, __shfl_xor_sync(0xffffffffu, best, m));
    if (lane == 0) {
      const int col = (prm.collided[n] != 0 || best <= 0.0) ? 1 : 0;
      prm.collided[n] = col;
      prm.fvel[2 * n] = col ? 0.0 : f_v[s][0];
      prm.fvel[2 * n + 1] = col ? 0.0 : f_v[s][1];
      if (out_collided) out_collided[q] = col;
      if (clearance) clearance[q] = (float)best;
      if constexpr (kEp) prm.ep_clear[q] = (float)best;
    }
  }
}

template <bool kMap>
__global__ void __launch_bounds__(32 * kWorldStepMaxWarps) world_step_kernel(const WorldParams prm, const WorldMapParams mp, const float* __restrict__ action,
                                                                           int32_t* __restrict__ out_collided, int32_t* __restrict__ out_arrived,
                                                                           float* __restrict__ clearance) {
  world_step_body<kMap, false, false>(prm, mp, WorldBlockParams{}, action, out_collided, out_arrived, clearance);
}

// episode mode: __maxnreg__(128) instead of __launch_bounds__(256), under which ptxas settles on 64 registers and spills (at most 8
// warps per CTA either way)
template <bool kMap>
__global__ void __maxnreg__(128) world_step_ep_kernel(const WorldParams prm, const WorldMapParams mp, const float* __restrict__ action,
                                                      int32_t* __restrict__ out_collided, int32_t* __restrict__ out_arrived,
                                                      float* __restrict__ clearance) {
  world_step_body<kMap, true, false>(prm, mp, WorldBlockParams{}, action, out_collided, out_arrived, clearance);
}

// Maps that block obstacles (nb_world_set_map_contact; always with maps): the obstacles move by world_move_obstacle_blocked.  kEp:
// episode mode.  __maxnreg__(128) as in world_step_ep_kernel: under __launch_bounds__(256) ptxas settles on 80 registers and spills.
template <bool kEp>
__global__ void __maxnreg__(128) world_step_block_kernel(const WorldParams prm, const WorldMapParams mp, const WorldBlockParams bp,
                                                                                 const float* __restrict__ action, int32_t* __restrict__ out_collided,
                                                                                 int32_t* __restrict__ out_arrived, float* __restrict__ clearance) {
  world_step_body<true, kEp, true>(prm, mp, bp, action, out_collided, out_arrived, clearance);
}

// Actuation limits and noise (nb_world_set_actuation): the step of any of the kernels above (kMap, kEp, kBlock; kMove false after
// world_contact_kernel) with the actuation stage.  __maxnreg__(128) as in world_step_ep_kernel.
template <bool kMap, bool kEp, bool kBlock, bool kMove>
__global__ void __maxnreg__(128) world_step_act_kernel(const WorldParams prm, const WorldMapParams mp, const WorldBlockParams bp, const WorldNoiseParams nz,
                                                       const float* __restrict__ action, int32_t* __restrict__ out_collided,
                                                       int32_t* __restrict__ out_arrived, float* __restrict__ clearance) {
  world_step_body<kMap, kEp, kBlock, kMove, true>(prm, mp, bp, action, out_collided, out_arrived, clearance, nz);
}

}  // namespace nb
