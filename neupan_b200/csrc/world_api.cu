// C ABI of the batched 2-D world (nb_world_*, include/neupan_b200.h): the host-side checks of configs, scenes, behaviours and fleets,
// the world handle, and the launches of the scan, rvo and step kernels.
#include <algorithm>
#include <cmath>
#include <new>
#include <vector>

#include "host_common.h"
#include "world_kernel.cuh"
#include "world_rvo_kernel.cuh"
#include "world_episode_kernel.cuh"

using nb::dalloc;
using nb::fail;

struct nb_world {
  nb_world_config cfg;
  int B = 0, O = 0, V = 0;
  int max_circ = 0, max_edges = 0, scan_threads = 0, scan_grid = 0;
  size_t scan_smem = 0;
  int32_t *d_obs_begin = nullptr, *d_vert_begin = nullptr, *d_slot = nullptr, *d_counts = nullptr, *d_kind = nullptr;
  int32_t *d_collided = nullptr, *d_arrived = nullptr;
  double *d_vertices = nullptr, *d_env = nullptr, *d_obs = nullptr, *d_states = nullptr;
  double* d_beam_cs = nullptr;  // (R, 2), fixed at creation
  // host copies of the scene (nb_world_set_behaviors checks against them)
  std::vector<int32_t> h_obs_begin, h_vert_begin, h_kind;
  std::vector<double> h_vertices, h_env;
  // obstacle behaviours (nb_world_set_behaviors; nb_world_set_scenes clears them): has_rvo false -> nb_world_step launches only
  // world_step_kernel
  bool has_rvo = false;
  uint64_t seed = 0;
  int rvo_cap = 0, rvo_grid = 0;
  size_t rvo_smem = 0;
  double *d_beh = nullptr, *d_rad = nullptr, *d_goal = nullptr;
  int32_t* d_draws = nullptr;
  int rvo_max_n = 0;  // the largest environment's obstacle count (rvo_cap = rvo_max_n + K)
  // robots per environment (nb_world_set_fleet; nb_world_set_scenes makes it 1, from the env rows): the per-robot arrays
  // (states, collided, arrived above, every robot's goal and the velocity of its last step) hold B K rows (world_set_robots)
  int K = 1;
  double *d_fgoal = nullptr, *d_fvel = nullptr;
  // robot types (nb_world_set_fleet_ex; type 0 is the config's robot): the table (T + 1 rows), each robot's type (B K, zeros
  // without a mix) and the largest environment's robot edge count (the scan's staging size; 0 with K = 1)
  nb::WorldRobotType* d_types = nullptr;
  int32_t* d_rtype = nullptr;
  int max_redges = 0;
  // host copies of the placed robots (nb_world_set_maps checks the start bodies against them): rows, types 1..T, each robot's type
  std::vector<double> h_robots;
  std::vector<nb_world_robot_type> h_types;
  std::vector<int32_t> h_rtype;
  // occupancy maps (nb_world_set_maps; nb_world_set_scenes(_ex) and nb_world_set_fleet(_ex) drop them): has_map false -> the
  // kernels' map-free instantiations
  bool has_map = false;
  nb::WorldMap* d_maps = nullptr;
  uint32_t* d_bits = nullptr;
  int32_t* d_env_map = nullptr;
  double window = 0.0;
  // host copies of the maps (nb_world_set_map_contact checks the obstacles' starts against them)
  std::vector<nb::WorldMap> h_maps;
  std::vector<uint32_t> h_bits;
  std::vector<int32_t> h_env_map;
  // maps that block obstacles (nb_world_set_map_contact; dropped with the maps and by nb_world_set_behaviors): has_block false -> the
  // kernels' instantiations without it
  bool has_block = false;
  int32_t *d_block = nullptr, *d_bounces = nullptr, *d_bounced = nullptr;
  // episode mode (nb_world_set_episodes; every other set call leaves it): ep_slots > 0 slots run the B = S scenes of the bank
  int ep_slots = 0, ep_max_steps = 0;
  int32_t *d_scene_of = nullptr, *d_live = nullptr, *d_reset = nullptr, *d_ep_t = nullptr, *d_ep_count = nullptr;  // count: next, finished
  float* d_ep_clear = nullptr;
  int32_t *d_r_col = nullptr, *d_r_arr = nullptr, *d_r_astep = nullptr, *d_r_end = nullptr, *d_r_reason = nullptr, *d_r_slot = nullptr;
  float* d_r_minclr = nullptr;
};

namespace {

// A convex polygon of n vertices (x0, y0, x1, y1, ...): every vertex off an edge lies strictly on the same side of it
// (rejects repeated and collinear vertices, reflex corners and self-intersecting stars).
bool world_convex(const double* v, int n) {
  double sign = 0.0;
  for (int k = 0; k < n; ++k) {
    const int k1 = (k + 1) % n;
    const double ex = v[2 * k1] - v[2 * k], ey = v[2 * k1 + 1] - v[2 * k + 1];
    for (int i = 0; i < n; ++i) {
      if (i == k || i == k1) continue;
      const double c = ex * (v[2 * i + 1] - v[2 * k + 1]) - ey * (v[2 * i] - v[2 * k]);
      if (!(c != 0.0) || (sign != 0.0 && (c > 0.0) != (sign > 0.0))) return false;
      sign = c;
    }
  }
  return true;
}

// Closed segments p-q and a-b intersect or touch (orientation tests; a zero orientation counts inside the other's bounding box).
bool world_segs_meet(const double* p, const double* q, const double* a, const double* b) {
  auto orient = [](const double* u, const double* v, const double* w) { return (v[0] - u[0]) * (w[1] - u[1]) - (v[1] - u[1]) * (w[0] - u[0]); };
  auto in_box = [](const double* u, const double* v, const double* w) {
    return std::min(u[0], v[0]) <= w[0] && w[0] <= std::max(u[0], v[0]) && std::min(u[1], v[1]) <= w[1] && w[1] <= std::max(u[1], v[1]);
  };
  const double d1 = orient(a, b, p), d2 = orient(a, b, q), d3 = orient(p, q, a), d4 = orient(p, q, b);
  if (((d1 > 0 && d2 < 0) || (d1 < 0 && d2 > 0)) && ((d3 > 0 && d4 < 0) || (d3 < 0 && d4 > 0))) return true;
  return (d1 == 0 && in_box(a, b, p)) || (d2 == 0 && in_box(a, b, q)) || (d3 == 0 && in_box(p, q, a)) || (d4 == 0 && in_box(p, q, b));
}

// Why the outline of n vertices (x0, y0, x1, y1, ...) is not a simple polygon, or nullptr when it is one: every edge has a length,
// the area is not zero, and no two non-adjacent edges intersect or touch.
const char* world_outline_problem(const double* v, int n) {
  double area2 = 0.0;
  for (int k = 0; k < n; ++k) {
    const int k1 = (k + 1) % n;
    if (v[2 * k] == v[2 * k1] && v[2 * k + 1] == v[2 * k1 + 1]) return "has a zero-length edge";
    area2 += v[2 * k] * v[2 * k1 + 1] - v[2 * k1] * v[2 * k + 1];
  }
  if (!(area2 != 0.0)) return "has zero area";
  for (int i = 0; i < n; ++i)
    for (int j = i + 2; j < n; ++j) {
      if (i == 0 && j == n - 1) continue;  // adjacent through the closing vertex
      if (world_segs_meet(v + 2 * i, v + 2 * ((i + 1) % n), v + 2 * j, v + 2 * ((j + 1) % n))) return "is not simple (two edges that do not share a vertex meet)";
    }
  return nullptr;
}

// a * b rounded on its own: the host compiler may not fuse it into a following sum (the device's dmul / dadd order)
double host_dmul(double a, double b) {
  volatile double p = a * b;
  return p;
}

bool world_finite(const double* a, size_t n) {
  for (size_t i = 0; i < n; ++i)
    if (!std::isfinite(a[i])) return false;
  return true;
}

int world_check_config(const nb_world_config* cfg) {
  if (!cfg) return fail(NB_ERR_INVALID, "nb_world: null config");
  if (cfg->kinematics < 0 || cfg->kinematics > 2) return fail(NB_ERR_INVALID, "kinematics currently only supports diff, acker or omni");
  if (cfg->num_beams < 1) return fail(NB_ERR_INVALID, "the lidar needs R >= 1 beams (got %d)", cfg->num_beams);
  if (cfg->max_envs < 1) return fail(NB_ERR_INVALID, "max_envs must be positive");
  if (!(cfg->step_time > 0) || !std::isfinite(cfg->step_time)) return fail(NB_ERR_INVALID, "step_time must be positive");
  if (cfg->kinematics == NB_KIN_ACKER && !(cfg->wheelbase > 0)) return fail(NB_ERR_INVALID, "acker needs a positive wheelbase");
  if (!(cfg->range_max > 0) || !std::isfinite(cfg->range_max)) return fail(NB_ERR_INVALID, "range_max must be positive and finite");
  if (!std::isfinite(cfg->angle_min) || !std::isfinite(cfg->angle_max) || !world_finite(cfg->scan_offset, 3))
    return fail(NB_ERR_INVALID, "lidar angles and scan_offset must be finite");
  const int nr = cfg->robot_num_vertices;
  if (nr < 3 || nr > nb::kWorldMaxVertices) return fail(NB_ERR_INVALID, "the robot polygon needs 3..%d vertices (got %d)", nb::kWorldMaxVertices, nr);
  if (!world_finite(cfg->robot_vertices, 2 * nr) || !world_convex(cfg->robot_vertices, nr)) return fail(NB_ERR_INVALID, "the robot polygon is not convex");
  return NB_OK;
}

// Every check of nb_world_set_scenes_ex, on the host (kind NULL: every obstacle is a circle or a convex polygon).  Fills the
// per-obstacle slots (circle rank / first edge index within the environment), the per-environment (circles, edges) counts and the
// largest counts of any environment when asked to.
int world_check_scenes(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obs, const int32_t* vert_begin,
                       const double* vertices, const double* envs, const int32_t* kind, std::vector<int32_t>* slot, std::vector<int32_t>* counts,
                       int* max_circ, int* max_edges) {
  if (int rc = world_check_config(cfg)) return rc;
  if (!obs_begin || !vert_begin || !envs) return fail(NB_ERR_INVALID, "nb_world scenes: null argument");
  if (B < 1 || B > cfg->max_envs) return fail(NB_ERR_INVALID, "B = %d outside [1, max_envs = %d]", B, cfg->max_envs);
  if (obs_begin[0] != 0) return fail(NB_ERR_INVALID, "obs_begin[0] must be 0");
  for (int b = 0; b < B; ++b) {
    const int n = obs_begin[b + 1] - obs_begin[b];
    if (n < 0) return fail(NB_ERR_INVALID, "obs_begin is not ascending at environment %d", b);
    if (n > nb::kWorldMaxObstacles) return fail(NB_ERR_INVALID, "environment %d has %d obstacles (at most %d)", b, n, nb::kWorldMaxObstacles);
  }
  const int O = obs_begin[B];
  if (O > 0 && !obs) return fail(NB_ERR_INVALID, "nb_world scenes: null obstacles");
  if (vert_begin[0] != 0) return fail(NB_ERR_INVALID, "vert_begin[0] must be 0");
  for (int o = 0; o < O; ++o) {
    const int nv = vert_begin[o + 1] - vert_begin[o];
    if (kind && kind[o] != 0) {
      if (kind[o] != 1) return fail(NB_ERR_INVALID, "obstacle %d has kind %d (0: circle or convex polygon, 1: outline)", o, kind[o]);
      if (nv < 3 || nv > nb::kWorldMaxOutlineVertices)
        return fail(NB_ERR_INVALID, "obstacle %d: an outline needs 3..%d vertices (got %d)", o, nb::kWorldMaxOutlineVertices, nv);
      continue;
    }
    if (nv != 0 && (nv < 3 || nv > nb::kWorldMaxVertices))
      return fail(NB_ERR_INVALID, "obstacle %d has %d vertices (0 for a circle, 3..%d for a polygon)", o, nv, nb::kWorldMaxVertices);
  }
  const int V = vert_begin[O];
  if (V > 0 && !vertices) return fail(NB_ERR_INVALID, "nb_world scenes: null vertices");
  if (!world_finite(envs, (size_t)B * nb::kWorldEnvCols) || !world_finite(obs, (size_t)O * nb::kWorldObsCols) || !world_finite(vertices, (size_t)V * 2))
    return fail(NB_ERR_INVALID, "nb_world scenes: non-finite value");
  if (slot) { slot->assign(O, 0); counts->assign(2 * (size_t)B, 0); *max_circ = 0; *max_edges = 0; }
  const double dt = cfg->step_time;
  for (int b = 0; b < B; ++b) {
    const double* e = envs + (size_t)nb::kWorldEnvCols * b;
    if (!(e[0] < e[2]) || !(e[1] < e[3])) return fail(NB_ERR_INVALID, "environment %d: the rectangle needs xmin < xmax and ymin < ymax", b);
    if (!(e[9] >= 0)) return fail(NB_ERR_INVALID, "environment %d: goal_threshold must be >= 0", b);
    int nc = 0, ne = 0;
    for (int o = obs_begin[b]; o < obs_begin[b + 1]; ++o) {
      const double* r = obs + (size_t)nb::kWorldObsCols * o;
      const int nv = vert_begin[o + 1] - vert_begin[o];
      if (nv == 0 && !(r[4] > 0)) return fail(NB_ERR_INVALID, "obstacle %d: a circle needs a positive radius", o);
      if (kind && kind[o] == 1) {
        if (const char* why = world_outline_problem(vertices + 2 * (size_t)vert_begin[o], nv)) return fail(NB_ERR_INVALID, "obstacle %d: the outline %s", o, why);
      } else if (nv > 0 && !world_convex(vertices + 2 * (size_t)vert_begin[o], nv)) {
        return fail(NB_ERR_INVALID, "obstacle %d is not a convex polygon", o);
      }
      for (int a = 0; a < 2; ++a) {
        if (r[2 + a] == 0.0) continue;
        const double lo = e[a], hi = e[2 + a];
        if (r[a] < lo || r[a] > hi) return fail(NB_ERR_INVALID, "obstacle %d moves but its centre starts outside the rectangle of environment %d", o, b);
        if (!(std::fabs(r[2 + a]) * dt < hi - lo)) return fail(NB_ERR_INVALID, "obstacle %d: |v| * step_time exceeds the rectangle of environment %d", o, b);
      }
      if (slot) (*slot)[o] = nv == 0 ? nc : ne;
      if (nv == 0) ++nc; else ne += nv;
    }
    // the scan stages an environment's edges in shared memory; 256 convex polygons cannot exceed this, outlines can
    if (ne > nb::kWorldMaxEdges) return fail(NB_ERR_INVALID, "environment %d has %d polygon edges (at most %d)", b, ne, nb::kWorldMaxEdges);
    if (slot) {
      (*counts)[2 * b] = nc; (*counts)[2 * b + 1] = ne;
      *max_circ = std::max(*max_circ, nc); *max_edges = std::max(*max_edges, ne);
    }
  }
  return NB_OK;
}

// Every check of nb_world_set_behaviors on the rows (kWorldBehCols) of valid scenes; obs holds the obstacles' current centres.
int world_check_behaviors(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obs, const double* envs,
                          const double* beh) {
  if (!beh) return fail(NB_ERR_INVALID, "nb_world behaviors: null behaviors");
  const double dt = cfg->step_time;
  for (int b = 0; b < B; ++b) {
    const double* e = envs + (size_t)nb::kWorldEnvCols * b;
    for (int o = obs_begin[b]; o < obs_begin[b + 1]; ++o) {
      const double* r = beh + (size_t)nb::kWorldBehCols * o;
      if (r[0] == 0.0) continue;  // constant velocity: the other columns are not read
      if (r[0] != 1.0) return fail(NB_ERR_INVALID, "obstacle %d has behaviour kind %g (0: constant velocity, 1: rvo)", o, r[0]);
      for (int c = 1; c < nb::kWorldBehCols; ++c)
        if (c != 7 && c != 8 && !std::isfinite(r[c])) return fail(NB_ERR_INVALID, "obstacle %d: behaviour column %d is not finite", o, c);
      const bool draw = std::isnan(r[7]) && std::isnan(r[8]);
      if (!draw && (!std::isfinite(r[7]) || !std::isfinite(r[8])))
        return fail(NB_ERR_INVALID, "obstacle %d: the goal must be finite, or NaN in both coordinates (drawn)", o);
      static const char* const names[] = {nullptr, "vxmax", "vymax", "acce", "factor", "speed", nullptr, nullptr, nullptr, "goal_threshold",
                                          "neighbor_range", "grid"};
      for (int c : {1, 2, 3, 4, 5, 9, 10, 11})
        if (!(r[c] > 0)) return fail(NB_ERR_INVALID, "obstacle %d: %s must be positive", o, names[c]);
      if (!(r[12] >= 0)) return fail(NB_ERR_INVALID, "obstacle %d: min_speed must be >= 0", o);
      if (r[6] != 0.0 && r[6] != 1.0) return fail(NB_ERR_INVALID, "obstacle %d: wander must be 0 or 1", o);
      for (int a = 0; a < 2; ++a) {
        const double span = 2.0 * std::min(r[3], r[1 + a]), n = std::ceil(span / r[11]);
        if (n > nb::kWorldRvoMaxAxis)
          return fail(NB_ERR_INVALID, "obstacle %d: up to %.0f candidate velocities on an axis (at most %d)", o, n, nb::kWorldRvoMaxAxis);
      }
      for (int a = 0; a < 2; ++a) {
        const double lo = e[a], hi = e[2 + a];
        if (obs[(size_t)nb::kWorldObsCols * o + a] < lo || obs[(size_t)nb::kWorldObsCols * o + a] > hi)
          return fail(NB_ERR_INVALID, "obstacle %d is reactive but its centre starts outside the rectangle of environment %d", o, b);
        if (!(r[1 + a] * dt < hi - lo)) return fail(NB_ERR_INVALID, "obstacle %d: %s * step_time exceeds the rectangle of environment %d", o, names[1 + a], b);
        if (!draw && (r[7 + a] < lo || r[7 + a] > hi)) return fail(NB_ERR_INVALID, "obstacle %d: its goal lies outside the rectangle of environment %d", o, b);
      }
    }
  }
  return NB_OK;
}

// Convex polygons (x0, y0, x1, y1, ...) overlap or touch: no edge normal of either separates their projections strictly (the step
// kernels' SAT, on the host).
bool world_bodies_meet(const double* a, int na, const double* b, int nb_) {
  for (int pass = 0; pass < 2; ++pass) {
    const double* p = pass ? b : a;
    const double* q = pass ? a : b;
    const int np = pass ? nb_ : na, nq = pass ? na : nb_;
    for (int k = 0; k < np; ++k) {
      const int k1 = (k + 1) % np;
      const double nx = -(p[2 * k1 + 1] - p[2 * k + 1]), ny = p[2 * k1] - p[2 * k];
      double pmin = INFINITY, pmax = -INFINITY, qmin = INFINITY, qmax = -INFINITY;
      for (int i = 0; i < np; ++i) { const double d = nx * p[2 * i] + ny * p[2 * i + 1]; pmin = std::min(pmin, d); pmax = std::max(pmax, d); }
      for (int i = 0; i < nq; ++i) { const double d = nx * q[2 * i] + ny * q[2 * i + 1]; qmin = std::min(qmin, d); qmax = std::max(qmax, d); }
      if (pmax < qmin || qmax < pmin) return false;
    }
  }
  return true;
}

// Type 0 (the robot of the config) and types 1..T as rows of the device type table; r is the circumradius about the state point
// (a reactive obstacle's neighbour circle), computed as the rvo kernel's products are rounded.
nb::WorldRobotType world_type_row(int32_t kinematics, int32_t nv, double L, const double* vertices) {
  nb::WorldRobotType t{};
  t.kinematics = kinematics; t.nv = nv; t.L = L;
  for (int i = 0; i < 2 * nv; ++i) t.v[i] = vertices[i];
  for (int k = 0; k < nv; ++k) t.r = std::max(t.r, std::sqrt(host_dmul(t.v[2 * k], t.v[2 * k]) + host_dmul(t.v[2 * k + 1], t.v[2 * k + 1])));
  return t;
}

std::vector<nb::WorldRobotType> world_type_table(const nb_world_config* cfg, int32_t T, const nb_world_robot_type* types) {
  std::vector<nb::WorldRobotType> table{world_type_row(cfg->kinematics, cfg->robot_num_vertices, cfg->wheelbase, cfg->robot_vertices)};
  for (int t = 0; t < T; ++t) table.push_back(world_type_row(types[t].kinematics, types[t].num_vertices, types[t].wheelbase, types[t].vertices));
  return table;
}

// Every check of nb_world_set_fleet_ex on the host: T in 0..kWorldMaxRobotTypes - 1 valid robot types (the checks the config's
// robot gets), K in 1..kWorldMaxFleet, finite rows, goal_threshold >= 0, every robot's type in 0..T, and no two robots of an
// environment whose bodies at their starts (each its own type's polygon) overlap or touch.  With T = 0 and no robot_type these are
// the checks and messages of nb_world_check_fleet.
int world_check_fleet(const nb_world_config* cfg, int32_t T, const nb_world_robot_type* types, int32_t B, int32_t K, const double* robots,
                      const int32_t* robot_type) {
  if (int rc = world_check_config(cfg)) return rc;
  if (T < 0 || T >= nb::kWorldMaxRobotTypes)
    return fail(NB_ERR_INVALID, "T = %d robot types besides type 0 (0..%d)", T, nb::kWorldMaxRobotTypes - 1);
  if (T > 0 && !types) return fail(NB_ERR_INVALID, "nb_world fleet: null types");
  for (int t = 1; t <= T; ++t) {
    const nb_world_robot_type& ty = types[t - 1];
    if (ty.kinematics < 0 || ty.kinematics > 2) return fail(NB_ERR_INVALID, "robot type %d: kinematics %d (diff, acker or omni)", t, ty.kinematics);
    if (ty.kinematics == NB_KIN_ACKER && !(ty.wheelbase > 0 && std::isfinite(ty.wheelbase)))
      return fail(NB_ERR_INVALID, "robot type %d: acker needs a positive wheelbase", t);
    const int nr = ty.num_vertices;
    if (nr < 3 || nr > nb::kWorldMaxVertices)
      return fail(NB_ERR_INVALID, "robot type %d: the polygon needs 3..%d vertices (got %d)", t, nb::kWorldMaxVertices, nr);
    if (!world_finite(ty.vertices, 2 * nr) || !world_convex(ty.vertices, nr)) return fail(NB_ERR_INVALID, "robot type %d: the polygon is not convex", t);
  }
  if (B < 1 || B > cfg->max_envs) return fail(NB_ERR_INVALID, "B = %d outside [1, max_envs = %d]", B, cfg->max_envs);
  if (K < 1 || K > nb::kWorldMaxFleet) return fail(NB_ERR_INVALID, "K = %d robots per environment (1..%d)", K, nb::kWorldMaxFleet);
  if (!robots) return fail(NB_ERR_INVALID, "nb_world fleet: null robots");
  for (int b = 0; b < B; ++b)
    for (int k = 0; k < K; ++k) {
      const double* r = robots + 6 * ((size_t)b * K + k);
      if (!world_finite(r, 6)) return fail(NB_ERR_INVALID, "environment %d, robot %d: non-finite value", b, k);
      if (!(r[5] >= 0)) return fail(NB_ERR_INVALID, "environment %d, robot %d: goal_threshold must be >= 0", b, k);
      if (robot_type) {
        const int t = robot_type[(size_t)b * K + k];
        if (t < 0 || t > T) return fail(NB_ERR_INVALID, "environment %d, robot %d: type %d outside 0..%d", b, k, t, T);
      }
    }
  const std::vector<nb::WorldRobotType> table = world_type_table(cfg, T, types);
  std::vector<double> body(2 * (size_t)K * nb::kWorldMaxVertices);
  std::vector<int> nv(K);
  for (int b = 0; b < B; ++b) {
    for (int k = 0; k < K; ++k) {
      const double* r = robots + 6 * ((size_t)b * K + k);
      const nb::WorldRobotType& ty = table[robot_type ? robot_type[(size_t)b * K + k] : 0];
      const double c = std::cos(r[2]), s = std::sin(r[2]);
      nv[k] = ty.nv;
      for (int v = 0; v < ty.nv; ++v) {
        const double px = ty.v[2 * v], py = ty.v[2 * v + 1];
        body[2 * ((size_t)k * nb::kWorldMaxVertices + v)] = r[0] + (c * px - s * py);
        body[2 * ((size_t)k * nb::kWorldMaxVertices + v) + 1] = r[1] + (s * px + c * py);
      }
    }
    for (int i = 0; i < K; ++i)
      for (int j = i + 1; j < K; ++j)
        if (world_bodies_meet(body.data() + 2 * (size_t)i * nb::kWorldMaxVertices, nv[i], body.data() + 2 * (size_t)j * nb::kWorldMaxVertices, nv[j]))
          return fail(NB_ERR_INVALID, "environment %d: the start bodies of robots %d and %d overlap", b, i, j);
  }
  return NB_OK;
}

// Grid line k of a map axis, rounded as the kernels round it (world_map_line), and the clamped floor index of world_map_floor.
double map_line(double lo, double r, int k) { return lo + host_dmul((double)k, r); }
int map_floor(double s, double lo, double r, int n) {
  const double f = std::floor((s - lo) / r);
  return f < -1.0 ? -1 : (f > (double)n ? n : (int)f);
}

// Every check of nb_world_set_maps on the host (robots NULL: without the start bodies).  Fills the device table when asked to.
int world_check_maps(const nb_world_config* cfg, int32_t T, const nb_world_robot_type* types, int32_t B, int32_t K, const double* robots,
                     const int32_t* robot_type, int32_t P, const nb_world_map* maps, const uint32_t* bits, const int32_t* env_map, double window,
                     std::vector<nb::WorldMap>* table) {
  if (robots) {
    if (int rc = world_check_fleet(cfg, T, types, B, K, robots, robot_type)) return rc;
  } else {
    if (int rc = world_check_config(cfg)) return rc;
    if (B < 1 || B > cfg->max_envs) return fail(NB_ERR_INVALID, "B = %d outside [1, max_envs = %d]", B, cfg->max_envs);
  }
  if (!maps || !bits || !env_map) return fail(NB_ERR_INVALID, "nb_world maps: null argument");
  if (P < 1 || P > cfg->max_envs) return fail(NB_ERR_INVALID, "P = %d maps outside [1, max_envs = %d]", P, cfg->max_envs);
  std::vector<nb::WorldMap> t(P);
  int64_t off = 0;
  for (int p = 0; p < P; ++p) {
    const nb_world_map& m = maps[p];
    if (m.width < 1 || m.width > nb::kWorldMaxMapSide || m.height < 1 || m.height > nb::kWorldMaxMapSide)
      return fail(NB_ERR_INVALID, "map %d: width %d and height %d must be in 1..%d", p, m.width, m.height, nb::kWorldMaxMapSide);
    if (!world_finite(m.origin, 2)) return fail(NB_ERR_INVALID, "map %d: the origin is not finite", p);
    if (!(std::isfinite(m.resolution) && m.resolution >= 0.01)) return fail(NB_ERR_INVALID, "map %d: the resolution must be finite and >= 0.01 m (got %g)", p, m.resolution);
    const int words = (m.width + 31) / 32;
    if (m.width % 32)
      for (int j = 0; j < m.height; ++j)
        if (bits[off + (int64_t)j * words + words - 1] >> (m.width % 32))
          return fail(NB_ERR_INVALID, "map %d: row %d has padding bits set past width %d", p, j, m.width);
    t[p] = nb::WorldMap{m.origin[0], m.origin[1], m.resolution, off, m.width, m.height, words, 0};
    off += (int64_t)m.height * words;
  }
  for (int b = 0; b < B; ++b)
    if (env_map[b] < -1 || env_map[b] >= P) return fail(NB_ERR_INVALID, "environment %d: map %d outside -1..%d", b, env_map[b], P - 1);
  if (!(window > 0.0 && window <= 10.0)) return fail(NB_ERR_INVALID, "window = %g outside (0, 10] m", window);
  if (robots) {  // no start body may overlap or touch an occupied cell (the fleet check's SAT and bodies)
    const std::vector<nb::WorldRobotType> tt = world_type_table(cfg, T, types);
    double body[2 * nb::kWorldMaxVertices];
    for (int b = 0; b < B; ++b) {
      if (env_map[b] < 0) continue;
      const nb::WorldMap& m = t[env_map[b]];
      for (int k = 0; k < K; ++k) {
        const double* r = robots + 6 * ((size_t)b * K + k);
        const nb::WorldRobotType& ty = tt[robot_type ? robot_type[(size_t)b * K + k] : 0];
        const double c = std::cos(r[2]), s = std::sin(r[2]);
        double xmin = INFINITY, xmax = -INFINITY, ymin = INFINITY, ymax = -INFINITY;
        for (int v = 0; v < ty.nv; ++v) {
          const double px = ty.v[2 * v], py = ty.v[2 * v + 1];
          body[2 * v] = r[0] + (c * px - s * py);
          body[2 * v + 1] = r[1] + (s * px + c * py);
          xmin = std::min(xmin, body[2 * v]); xmax = std::max(xmax, body[2 * v]);
          ymin = std::min(ymin, body[2 * v + 1]); ymax = std::max(ymax, body[2 * v + 1]);
        }
        const int i0 = std::max(map_floor(xmin, m.x0, m.r, m.W) - 1, 0), i1 = std::min(map_floor(xmax, m.x0, m.r, m.W) + 1, m.W - 1);
        const int j0 = std::max(map_floor(ymin, m.y0, m.r, m.H) - 1, 0), j1 = std::min(map_floor(ymax, m.y0, m.r, m.H) + 1, m.H - 1);
        for (int j = j0; j <= j1; ++j)
          for (int i = i0; i <= i1; ++i) {
            if (!((bits[m.off + (int64_t)j * m.words + (i >> 5)] >> (i & 31)) & 1u)) continue;
            const double xa = map_line(m.x0, m.r, i), xb = map_line(m.x0, m.r, i + 1), ya = map_line(m.y0, m.r, j), yb = map_line(m.y0, m.r, j + 1);
            const double cell[8] = {xa, ya, xb, ya, xb, yb, xa, yb};
            if (world_bodies_meet(body, ty.nv, cell, 4))
              return fail(NB_ERR_INVALID, "environment %d, robot %d: the start body overlaps or touches occupied cell (%d, %d) of map %d", b, k, i, j, env_map[b]);
          }
      }
    }
  }
  if (table) *table = std::move(t);
  return NB_OK;
}

// Frees the map-contact arrays: obstacles pass over the maps from here on.
void world_drop_contact(nb_world* w) {
  void* old[] = {w->d_block, w->d_bounces, w->d_bounced};
  for (void* p : old)
    if (p) cudaFree(p);
  w->d_block = w->d_bounces = w->d_bounced = nullptr;
  w->has_block = false;
}

// Frees the maps (and their contact flags): the kernels' map-free instantiations from here on.
void world_drop_maps(nb_world* w) {
  void* old[] = {w->d_maps, w->d_bits, w->d_env_map};
  for (void* p : old)
    if (p) cudaFree(p);
  w->d_maps = nullptr; w->d_bits = nullptr; w->d_env_map = nullptr;
  w->has_map = false;
  w->h_maps.clear(); w->h_bits.clear(); w->h_env_map.clear();
  world_drop_contact(w);
}

// Does the footprint of obstacle o at its centre (row) overlap or touch cell [xa, xb] x [ya, yb]?  The host's reading of the
// kernels' contact test: a circle by its centre's distance to the closed cell, a convex polygon by SAT, an outline by its edges,
// its vertex 0 in the cell or the cell's corner in it.
bool world_footprint_meets_cell(const double* row, const double* rel, int nv, int kind, double xa, double ya, double xb, double yb) {
  const double cell[8] = {xa, ya, xb, ya, xb, yb, xa, yb};
  if (nv == 0) {
    const double dx = std::max({xa - row[0], 0.0, row[0] - xb}), dy = std::max({ya - row[1], 0.0, row[1] - yb});
    return std::sqrt(dx * dx + dy * dy) <= row[4];
  }
  double v[2 * nb::kWorldMaxOutlineVertices];
  for (int k = 0; k < nv; ++k) { v[2 * k] = row[0] + rel[2 * k]; v[2 * k + 1] = row[1] + rel[2 * k + 1]; }
  if (kind == 0) return world_bodies_meet(v, nv, cell, 4);
  bool in = false;  // even-odd test of the cell's corner (xa, ya) against the outline
  for (int k = 0; k < nv; ++k) {
    const int k1 = (k + 1) % nv;
    for (int e = 0; e < 4; ++e)
      if (world_segs_meet(v + 2 * k, v + 2 * k1, cell + 2 * e, cell + 2 * ((e + 1) % 4))) return true;
    const double ax = v[2 * k], ay = v[2 * k + 1], bx = v[2 * k1], by = v[2 * k1 + 1];
    if ((ay > ya) != (by > ya) && xa < ax + (ya - ay) * (bx - ax) / (by - ay)) in = !in;
  }
  return in || (xa <= v[0] && v[0] <= xb && ya <= v[1] && v[1] <= yb);
}

// Every check of nb_world_set_map_contact on valid scenes, behaviours (NULL: every obstacle constant) and maps (the device table
// and its bits); obs holds the obstacles' current centres and velocities.
int world_check_contact(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obs, const int32_t* vert_begin,
                        const double* vertices, const int32_t* kind, const double* beh, const std::vector<nb::WorldMap>& maps, const uint32_t* bits,
                        const int32_t* env_map, const int32_t* flags) {
  if (!flags) return fail(NB_ERR_INVALID, "nb_world map contact: null flags");
  const double dt = cfg->step_time;
  for (int b = 0; b < B; ++b) {
    if (flags[b] != 0 && flags[b] != 1) return fail(NB_ERR_INVALID, "environment %d: map contact flag %d (0 or 1)", b, flags[b]);
    if (flags[b] == 0) continue;
    if (env_map[b] < 0) return fail(NB_ERR_INVALID, "environment %d: its map blocks obstacles but it has no map", b);
    const nb::WorldMap& m = maps[env_map[b]];
    for (int o = obs_begin[b]; o < obs_begin[b + 1]; ++o) {
      const double* row = obs + (size_t)nb::kWorldObsCols * o;
      const double* br = beh ? beh + (size_t)nb::kWorldBehCols * o : nullptr;
      const bool reactive = br && br[0] == 1.0;
      if (!reactive && row[2] == 0.0 && row[3] == 0.0) continue;  // static obstacles may overlap walls
      const double top = reactive ? std::sqrt(br[1] * br[1] + br[2] * br[2]) : std::sqrt(row[2] * row[2] + row[3] * row[3]);
      if (!(top * dt < m.r))
        return fail(NB_ERR_INVALID, "environment %d, obstacle %d: top speed %g m/s * step_time = %g m is not below the map's resolution %g m", b, o,
                    top, top * dt, m.r);
      const int v0 = vert_begin[o], nv = vert_begin[o + 1] - v0;
      const double* rel = vertices + 2 * (size_t)v0;
      double xmin = row[0] - row[4], xmax = row[0] + row[4], ymin = row[1] - row[4], ymax = row[1] + row[4];
      if (nv > 0) {
        xmin = ymin = INFINITY; xmax = ymax = -INFINITY;
        for (int k = 0; k < nv; ++k) {
          xmin = std::min(xmin, row[0] + rel[2 * k]); xmax = std::max(xmax, row[0] + rel[2 * k]);
          ymin = std::min(ymin, row[1] + rel[2 * k + 1]); ymax = std::max(ymax, row[1] + rel[2 * k + 1]);
        }
      }
      const int i0 = std::max(map_floor(xmin, m.x0, m.r, m.W) - 1, 0), i1 = std::min(map_floor(xmax, m.x0, m.r, m.W) + 1, m.W - 1);
      const int j0 = std::max(map_floor(ymin, m.y0, m.r, m.H) - 1, 0), j1 = std::min(map_floor(ymax, m.y0, m.r, m.H) + 1, m.H - 1);
      for (int j = j0; j <= j1; ++j)
        for (int i = i0; i <= i1; ++i) {
          if (!((bits[m.off + (int64_t)j * m.words + (i >> 5)] >> (i & 31)) & 1u)) continue;
          if (world_footprint_meets_cell(row, rel, nv, kind ? kind[o] : 0, map_line(m.x0, m.r, i), map_line(m.y0, m.r, j), map_line(m.x0, m.r, i + 1),
                                         map_line(m.y0, m.r, j + 1)))
            return fail(NB_ERR_INVALID, "environment %d, obstacle %d: moves but its start footprint overlaps or touches occupied cell (%d, %d) of map %d",
                        b, o, i, j, env_map[b]);
        }
    }
  }
  return NB_OK;
}

// Leaves episode mode: frees the slot and result arrays (the scenes' own rows stay as they are).
void world_drop_episodes(nb_world* w) {
  void* old[] = {w->d_scene_of, w->d_live, w->d_reset, w->d_ep_t, w->d_ep_count, w->d_ep_clear, w->d_r_col, w->d_r_arr, w->d_r_astep,
                 w->d_r_end, w->d_r_reason, w->d_r_slot, w->d_r_minclr};
  for (void* p : old)
    if (p) cudaFree(p);
  w->d_scene_of = w->d_live = w->d_reset = w->d_ep_t = w->d_ep_count = nullptr;
  w->d_r_col = w->d_r_arr = w->d_r_astep = w->d_r_end = w->d_r_reason = w->d_r_slot = nullptr;
  w->d_ep_clear = w->d_r_minclr = nullptr;
  w->ep_slots = 0; w->ep_max_steps = 0;
}

// Every check of nb_world_set_episodes on the host: S in 1..max_envs, slots in 1..S, max_steps >= 1, and (robot_type not NULL)
// robot k of every scene of the type of robot k of scene 0.
int world_check_episodes(const nb_world_config* cfg, int32_t S, int32_t K, const int32_t* robot_type, int32_t slots, int32_t max_steps) {
  if (int rc = world_check_config(cfg)) return rc;
  if (S < 1 || S > cfg->max_envs) return fail(NB_ERR_INVALID, "a bank of S = %d scenes outside [1, max_envs = %d]", S, cfg->max_envs);
  if (K < 1 || K > nb::kWorldMaxFleet) return fail(NB_ERR_INVALID, "K = %d robots per scene (1..%d)", K, nb::kWorldMaxFleet);
  if (slots < 1 || slots > S) return fail(NB_ERR_INVALID, "slots = %d outside [1, S = %d]", slots, S);
  if (max_steps < 1) return fail(NB_ERR_INVALID, "max_steps = %d must be >= 1", max_steps);
  if (robot_type)
    for (int s = 1; s < S; ++s)
      for (int k = 0; k < K; ++k)
        if (robot_type[(size_t)s * K + k] != robot_type[k])
          return fail(NB_ERR_INVALID, "scene %d, robot %d: type %d but robot %d of scene 0 has type %d (a robot keeps its type in every scene of a bank)",
                      s, k, robot_type[(size_t)s * K + k], k, robot_type[k]);
  return NB_OK;
}

nb::WorldMapParams world_map_params(const nb_world* w) { return nb::WorldMapParams{w->d_maps, w->d_bits, w->d_env_map, w->window}; }
nb::WorldBlockParams world_block_params(const nb_world* w) { return nb::WorldBlockParams{w->d_block, w->d_bounces, w->d_bounced}; }

template <bool kMap>
int world_scan_occupancy(nb_world* w, int* per_sm) {
  // the occupancy query sees the kernel's current limit; nb_world_scan sets it again before every launch
  NB_CUDA(cudaFuncSetAttribute(nb::world_scan_kernel<kMap, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(w->scan_smem, 1)));
  NB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, nb::world_scan_kernel<kMap, false>, w->scan_threads, w->scan_smem));
  return NB_OK;
}

// scan launch shape: the largest environment's circles and edges (and with K > 1 the K robot bodies) in shared memory, one thread
// per beam of the environment's K R beams (at most 256); the instantiation with maps when the handle has any
int world_scan_shape(nb_world* w, int B) {
  const int nre = w->K > 1 ? w->max_redges : 0;
  w->scan_smem = (size_t)w->max_circ * (3 * sizeof(double) + sizeof(int32_t)) + (size_t)w->max_edges * (4 * sizeof(double) + sizeof(int32_t)) +
                 (size_t)nre * (4 * sizeof(double) + sizeof(int32_t));
  w->scan_threads = std::min(256, std::max(32, (w->K * w->cfg.num_beams + 31) / 32 * 32));
  int per_sm = 0, sms = 0;
  if (int rc = w->has_map ? world_scan_occupancy<true>(w, &per_sm) : world_scan_occupancy<false>(w, &per_sm)) return rc;
  NB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, w->cfg.device));
  if (per_sm < 1) return fail(NB_ERR_CUDA, "world_scan_kernel: %zu B of shared memory do not fit", w->scan_smem);
  w->scan_grid = std::min(B, per_sm * sms);
  return NB_OK;
}

// rvo launch shape: the largest environment's rows (+ the K robots) and one cone list per warp in shared memory
int world_rvo_shape(nb_world* w, int B) {
  w->rvo_cap = w->rvo_max_n + w->K;
  w->rvo_smem = (size_t)w->rvo_cap * (5 * sizeof(double) + nb::kWorldRvoWarps * (6 * sizeof(double) + sizeof(int32_t)));
  NB_CUDA(cudaFuncSetAttribute(nb::world_rvo_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)w->rvo_smem));
  int per_sm = 0, sms = 0;
  NB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, nb::world_rvo_kernel<false>, 32 * nb::kWorldRvoWarps, w->rvo_smem));
  NB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, w->cfg.device));
  if (per_sm < 1) return fail(NB_ERR_CUDA, "world_rvo_kernel: %zu B of shared memory do not fit", w->rvo_smem);
  w->rvo_grid = std::min(B, per_sm * sms);
  return NB_OK;
}

// (Re)allocates the per-robot arrays for B K robots and uploads the rows [start x, y, theta, goal x, y, threshold] (robot k of
// environment b at row b K + k): every robot at its start, flags and velocities cleared.  The type table is type 0 and types[0 .. T);
// robot_type NULL: every robot is type 0.
int world_set_robots(nb_world* w, int B, int K, const double* robots, int T, const nb_world_robot_type* types, const int32_t* robot_type) {
  const size_t N = (size_t)B * K;
  std::vector<double> states(3 * N), goal(3 * N);
  for (size_t n = 0; n < N; ++n)
    for (int c = 0; c < 3; ++c) { states[3 * n + c] = robots[6 * n + c]; goal[3 * n + c] = robots[6 * n + 3 + c]; }
  const std::vector<nb::WorldRobotType> table = world_type_table(&w->cfg, T, types);
  std::vector<int32_t> rtype(N, 0);
  if (robot_type) rtype.assign(robot_type, robot_type + N);
  int max_redges = 0;
  for (int b = 0; K > 1 && b < B; ++b) {
    int e = 0;
    for (int k = 0; k < K; ++k) e += table[rtype[(size_t)b * K + k]].nv;
    max_redges = std::max(max_redges, e);
  }
  void* old[] = {w->d_states, w->d_collided, w->d_arrived, w->d_fgoal, w->d_fvel, w->d_types, w->d_rtype};
  for (void* p : old)
    if (p) cudaFree(p);
  w->d_states = w->d_fgoal = w->d_fvel = nullptr;
  w->d_collided = w->d_arrived = w->d_rtype = nullptr;
  w->d_types = nullptr;
  NB_CUDA(dalloc(&w->d_states, 3 * N));
  NB_CUDA(dalloc(&w->d_collided, N));
  NB_CUDA(dalloc(&w->d_arrived, N));
  NB_CUDA(dalloc(&w->d_fgoal, 3 * N));
  NB_CUDA(dalloc(&w->d_fvel, 2 * N));
  NB_CUDA(dalloc(&w->d_types, table.size()));
  NB_CUDA(dalloc(&w->d_rtype, N));
  NB_CUDA(cudaMemcpy(w->d_states, states.data(), sizeof(double) * 3 * N, cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(w->d_fgoal, goal.data(), sizeof(double) * 3 * N, cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(w->d_types, table.data(), sizeof(nb::WorldRobotType) * table.size(), cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(w->d_rtype, rtype.data(), sizeof(int32_t) * N, cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemset(w->d_collided, 0, sizeof(int32_t) * N));
  NB_CUDA(cudaMemset(w->d_arrived, 0, sizeof(int32_t) * N));
  NB_CUDA(cudaMemset(w->d_fvel, 0, sizeof(double) * 2 * N));
  w->K = K;
  w->max_redges = max_redges;
  w->h_robots.assign(robots, robots + 6 * N);
  w->h_types.assign(types, types + T);
  w->h_rtype = rtype;
  return NB_OK;
}

nb::WorldParams world_params(const nb_world* w) {
  nb::WorldParams prm;
  const nb_world_config& c = w->cfg;
  prm.B = w->ep_slots ? w->ep_slots : w->B; prm.R = c.num_beams;
  prm.dt = c.step_time; prm.range_max = c.range_max; prm.beam_cs = w->d_beam_cs;
  prm.off_x = c.scan_offset[0]; prm.off_y = c.scan_offset[1]; prm.off_th = c.scan_offset[2];
  prm.types = w->d_types; prm.rtype = w->d_rtype;
  prm.obs_begin = w->d_obs_begin; prm.vert_begin = w->d_vert_begin; prm.slot = w->d_slot; prm.counts = w->d_counts; prm.kind = w->d_kind;
  prm.vertices = w->d_vertices; prm.env = w->d_env; prm.obs = w->d_obs; prm.states = w->d_states;
  prm.collided = w->d_collided; prm.arrived = w->d_arrived;
  prm.K = w->K; prm.fgoal = w->d_fgoal; prm.fvel = w->d_fvel;
  prm.scene_of = w->d_scene_of; prm.live = w->d_live; prm.ep_clear = w->d_ep_clear;
  return prm;
}

// per_robot: the count argument is the robot count N = B K (B itself with one robot per environment), in episode mode the slot
// robots slots K; otherwise (the obstacle-side calls) the environment count B (S in episode mode)
int world_ready(const nb_world* w, int32_t B, const char* what, bool per_robot = false) {
  if (!w) return fail(NB_ERR_INVALID, "%s: null handle", what);
  if (!w->B) return fail(NB_ERR_INVALID, "%s: no scenes set (nb_world_set_scenes)", what);
  if (per_robot && w->ep_slots) {
    if (B != w->ep_slots * w->K)
      return fail(NB_ERR_INVALID, "%s: count = %d but the world runs episodes in %d slots x %d robots (N = %d)", what, B, w->ep_slots, w->K,
                  w->ep_slots * w->K);
    return NB_OK;
  }
  if (per_robot && w->K > 1) {
    if (B != w->B * w->K)
      return fail(NB_ERR_INVALID, "%s: count = %d but the world has %d environments x %d robots (N = %d)", what, B, w->B, w->K, w->B * w->K);
    return NB_OK;
  }
  if (B != w->B) return fail(NB_ERR_INVALID, "%s: B = %d but the scenes were set for %d environments", what, B, w->B);
  return NB_OK;
}

nb::WorldRvoParams world_rvo_params(const nb_world* w, const float* action) {
  nb::WorldRvoParams rp;
  rp.beh = w->d_beh; rp.radius = w->d_rad; rp.goal = w->d_goal; rp.draws = w->d_draws; rp.action = action;
  rp.seed = w->seed; rp.cap = w->rvo_cap;
  return rp;
}

}  // namespace

extern "C" {

int nb_world_create(const nb_world_config* cfg, nb_world_t** out) {
  if (!out) return fail(NB_ERR_INVALID, "nb_world_create: null argument");
  *out = nullptr;
  if (int rc = world_check_config(cfg)) return rc;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || cfg->device < 0 || cfg->device >= ndev)
    return fail(NB_ERR_NO_DEVICE, "no CUDA device available: neupan_b200 has no CPU fallback");
  NB_CUDA(cudaSetDevice(cfg->device));
  nb_world* w = new (std::nothrow) nb_world();
  if (!w) return fail(NB_ERR_INVALID, "out of host memory");
  w->cfg = *cfg;
  // cos / sin of the beam angles a_i = numpy.linspace(angle_min, angle_max, R)[i] (i * step + start, the last one = stop)
  const int R = cfg->num_beams;
  const double step = R > 1 ? (cfg->angle_max - cfg->angle_min) / (double)(R - 1) : 0.0;
  std::vector<double> cs(2 * (size_t)R);
  for (int i = 0; i < R; ++i) {
    const double a = R == 1 ? cfg->angle_min : (i == R - 1 ? cfg->angle_max : (double)i * step + cfg->angle_min);
    cs[2 * i] = std::cos(a);
    cs[2 * i + 1] = std::sin(a);
  }
  cudaError_t e = dalloc(&w->d_beam_cs, cs.size());
  if (e == cudaSuccess) e = cudaMemcpy(w->d_beam_cs, cs.data(), sizeof(double) * cs.size(), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    nb_world_destroy(w);
    return fail(NB_ERR_CUDA, "nb_world_create: %s", cudaGetErrorString(e));
  }
  *out = w;
  return NB_OK;
}

int nb_world_destroy(nb_world_t* w) {
  if (!w) return NB_OK;
  cudaSetDevice(w->cfg.device);
  world_drop_episodes(w);
  void* bufs[] = {w->d_obs_begin, w->d_vert_begin, w->d_slot, w->d_counts, w->d_kind, w->d_collided, w->d_arrived, w->d_vertices, w->d_env, w->d_obs,
                  w->d_states, w->d_beam_cs, w->d_beh, w->d_rad, w->d_goal, w->d_draws, w->d_fgoal, w->d_fvel, w->d_types, w->d_rtype,
                  w->d_maps, w->d_bits, w->d_env_map, w->d_block, w->d_bounces, w->d_bounced};
  for (void* b : bufs)
    if (b) cudaFree(b);
  delete w;
  return NB_OK;
}

int nb_world_check_scenes_ex(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obstacles, const int32_t* vert_begin,
                             const double* vertices, const double* envs, const int32_t* obs_kind) {
  return world_check_scenes(cfg, B, obs_begin, obstacles, vert_begin, vertices, envs, obs_kind, nullptr, nullptr, nullptr, nullptr);
}

int nb_world_check_scenes(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obstacles, const int32_t* vert_begin,
                          const double* vertices, const double* envs) {
  return nb_world_check_scenes_ex(cfg, B, obs_begin, obstacles, vert_begin, vertices, envs, nullptr);
}

int nb_world_set_scenes_ex(nb_world_t* w, int32_t B, const int32_t* obs_begin, const double* obstacles, const int32_t* vert_begin,
                           const double* vertices, const double* envs, const int32_t* obs_kind) {
  if (!w) return fail(NB_ERR_INVALID, "nb_world_set_scenes: null handle");
  std::vector<int32_t> slot, counts;
  int max_circ = 0, max_edges = 0;
  if (int rc = world_check_scenes(&w->cfg, B, obs_begin, obstacles, vert_begin, vertices, envs, obs_kind, &slot, &counts, &max_circ, &max_edges))
    return rc;
  const int O = obs_begin[B], V = vert_begin[O];
  std::vector<double> robots(6 * (size_t)B);  // one robot per environment until nb_world_set_fleet: the env rows' start and goal
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < 6; ++c) robots[6 * (size_t)b + c] = envs[(size_t)nb::kWorldEnvCols * b + 4 + c];
  NB_CUDA(cudaSetDevice(w->cfg.device));
  void* old[] = {w->d_obs_begin, w->d_vert_begin, w->d_slot, w->d_counts, w->d_kind, w->d_vertices, w->d_env, w->d_obs,
                 w->d_beh, w->d_rad, w->d_goal, w->d_draws};
  for (void* b : old)
    if (b) cudaFree(b);
  w->d_obs_begin = w->d_vert_begin = w->d_slot = w->d_counts = w->d_kind = w->d_draws = nullptr;
  w->d_vertices = w->d_env = w->d_obs = w->d_beh = w->d_rad = w->d_goal = nullptr;
  w->B = 0;
  w->has_rvo = false;  // new scenes: every obstacle keeps a constant velocity until nb_world_set_behaviors
  world_drop_maps(w);  // and has no map until nb_world_set_maps
  world_drop_episodes(w);  // and runs as a plain world until nb_world_set_episodes
  w->h_obs_begin.assign(obs_begin, obs_begin + B + 1);
  w->h_vert_begin.assign(vert_begin, vert_begin + O + 1);
  w->h_vertices.assign(vertices, vertices + 2 * (size_t)V);
  if (obs_kind) w->h_kind.assign(obs_kind, obs_kind + O);
  else w->h_kind.assign(O, 0);
  w->h_env.assign(envs, envs + (size_t)nb::kWorldEnvCols * B);
  NB_CUDA(dalloc(&w->d_obs_begin, (size_t)B + 1));
  NB_CUDA(dalloc(&w->d_vert_begin, (size_t)O + 1));
  NB_CUDA(dalloc(&w->d_slot, (size_t)O));
  NB_CUDA(dalloc(&w->d_counts, 2 * (size_t)B));
  NB_CUDA(dalloc(&w->d_kind, (size_t)O));
  if (O && obs_kind) NB_CUDA(cudaMemcpy(w->d_kind, obs_kind, sizeof(int32_t) * O, cudaMemcpyHostToDevice));
  else if (O) NB_CUDA(cudaMemset(w->d_kind, 0, sizeof(int32_t) * O));
  NB_CUDA(dalloc(&w->d_vertices, 2 * (size_t)V));
  NB_CUDA(dalloc(&w->d_env, (size_t)nb::kWorldEnvCols * B));
  NB_CUDA(dalloc(&w->d_obs, (size_t)nb::kWorldObsCols * O));
  NB_CUDA(cudaMemcpy(w->d_obs_begin, obs_begin, sizeof(int32_t) * (B + 1), cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(w->d_vert_begin, vert_begin, sizeof(int32_t) * (O + 1), cudaMemcpyHostToDevice));
  if (O) NB_CUDA(cudaMemcpy(w->d_slot, slot.data(), sizeof(int32_t) * O, cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(w->d_counts, counts.data(), sizeof(int32_t) * 2 * B, cudaMemcpyHostToDevice));
  if (V) NB_CUDA(cudaMemcpy(w->d_vertices, vertices, sizeof(double) * 2 * V, cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(w->d_env, envs, sizeof(double) * nb::kWorldEnvCols * B, cudaMemcpyHostToDevice));
  if (O) NB_CUDA(cudaMemcpy(w->d_obs, obstacles, sizeof(double) * nb::kWorldObsCols * O, cudaMemcpyHostToDevice));
  if (int rc = world_set_robots(w, B, 1, robots.data(), 0, nullptr, nullptr)) return rc;
  w->max_circ = max_circ; w->max_edges = max_edges;
  if (int rc = world_scan_shape(w, B)) return rc;
  w->B = B; w->O = O; w->V = V;
  NB_CUDA(cudaDeviceSynchronize());
  return NB_OK;
}

int nb_world_set_scenes(nb_world_t* w, int32_t B, const int32_t* obs_begin, const double* obstacles, const int32_t* vert_begin,
                        const double* vertices, const double* envs) {
  return nb_world_set_scenes_ex(w, B, obs_begin, obstacles, vert_begin, vertices, envs, nullptr);
}

int nb_world_check_behaviors(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obstacles, const int32_t* vert_begin,
                             const double* vertices, const double* envs, const int32_t* obs_kind, const double* behaviors, uint64_t seed) {
  (void)seed;  // every seed is valid: drawn goals lie in the rectangle by construction
  if (int rc = world_check_scenes(cfg, B, obs_begin, obstacles, vert_begin, vertices, envs, obs_kind, nullptr, nullptr, nullptr, nullptr)) return rc;
  return world_check_behaviors(cfg, B, obs_begin, obstacles, envs, behaviors);
}

int nb_world_set_behaviors(nb_world_t* w, int32_t B, const double* behaviors, uint64_t seed) {
  if (int rc = world_ready(w, B, "nb_world_set_behaviors")) return rc;
  NB_CUDA(cudaSetDevice(w->cfg.device));
  const int O = w->O;
  std::vector<double> obs((size_t)nb::kWorldObsCols * O);
  if (O) NB_CUDA(cudaMemcpy(obs.data(), w->d_obs, sizeof(double) * obs.size(), cudaMemcpyDeviceToHost));  // the current centres
  if (int rc = world_check_behaviors(&w->cfg, B, w->h_obs_begin.data(), obs.data(), w->h_env.data(), behaviors)) return rc;
  world_drop_episodes(w);
  world_drop_contact(w);  // which obstacles move has changed: the contact flags need their checks again
  // radii (circle: its own; polygon: the largest vertex norm), initial goals (NaN: draw 0) and draw counters
  std::vector<double> rad(O), goal(2 * (size_t)O, 0.0);
  std::vector<int32_t> draws(O, 0);
  bool any = false;
  int max_n = 0;
  for (int b = 0; b < B; ++b) {
    const int o0 = w->h_obs_begin[b], o1 = w->h_obs_begin[b + 1];
    const double* e = w->h_env.data() + (size_t)nb::kWorldEnvCols * b;
    max_n = std::max(max_n, o1 - o0);
    for (int o = o0; o < o1; ++o) {
      const int v0 = w->h_vert_begin[o], v1 = w->h_vert_begin[o + 1];
      double r = v0 == v1 ? obs[(size_t)nb::kWorldObsCols * o + 4] : 0.0;
      for (int k = v0; k < v1; ++k) {
        const double x = w->h_vertices[2 * k], y = w->h_vertices[2 * k + 1];
        r = std::max(r, std::sqrt(host_dmul(x, x) + host_dmul(y, y)));
      }
      rad[o] = r;
      const double* row = behaviors + (size_t)nb::kWorldBehCols * o;
      if (row[0] != 1.0) continue;
      any = true;
      if (std::isnan(row[7])) {
        const uint64_t key = nb::world_rvo_key(seed, b, o - o0);
        goal[2 * o] = e[0] + host_dmul(nb::world_u01(nb::splitmix64_at(key, 0)), e[2] - e[0]);  // draw 0
        goal[2 * o + 1] = e[1] + host_dmul(nb::world_u01(nb::splitmix64_at(key, 1)), e[3] - e[1]);
        draws[o] = 1;
      } else {
        goal[2 * o] = row[7]; goal[2 * o + 1] = row[8];
      }
    }
  }
  void* old[] = {w->d_beh, w->d_rad, w->d_goal, w->d_draws};
  for (void* p : old)
    if (p) cudaFree(p);
  w->d_beh = w->d_rad = w->d_goal = nullptr;
  w->d_draws = nullptr;
  w->has_rvo = false;
  NB_CUDA(dalloc(&w->d_beh, (size_t)nb::kWorldBehCols * O));
  NB_CUDA(dalloc(&w->d_rad, (size_t)O));
  NB_CUDA(dalloc(&w->d_goal, 2 * (size_t)O));
  NB_CUDA(dalloc(&w->d_draws, (size_t)O));
  if (O) {
    NB_CUDA(cudaMemcpy(w->d_beh, behaviors, sizeof(double) * nb::kWorldBehCols * O, cudaMemcpyHostToDevice));
    NB_CUDA(cudaMemcpy(w->d_rad, rad.data(), sizeof(double) * O, cudaMemcpyHostToDevice));
    NB_CUDA(cudaMemcpy(w->d_goal, goal.data(), sizeof(double) * 2 * O, cudaMemcpyHostToDevice));
    NB_CUDA(cudaMemcpy(w->d_draws, draws.data(), sizeof(int32_t) * O, cudaMemcpyHostToDevice));
  }
  w->seed = seed;
  w->rvo_max_n = max_n;
  if (int rc = world_rvo_shape(w, B)) return rc;
  w->has_rvo = any;
  NB_CUDA(cudaDeviceSynchronize());
  return NB_OK;
}

int nb_world_read_behaviors(nb_world_t* w, int32_t B, double* goals, int32_t* draws, void* stream) {
  if (int rc = world_ready(w, B, "nb_world_read_behaviors")) return rc;
  if (!w->d_goal) return fail(NB_ERR_INVALID, "nb_world_read_behaviors: no behaviours set (nb_world_set_behaviors)");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  if (goals && w->O) NB_CUDA(cudaMemcpyAsync(goals, w->d_goal, sizeof(double) * 2 * w->O, cudaMemcpyDeviceToDevice, st));
  if (draws && w->O) NB_CUDA(cudaMemcpyAsync(draws, w->d_draws, sizeof(int32_t) * w->O, cudaMemcpyDeviceToDevice, st));
  return NB_OK;
}

int nb_world_scan(nb_world_t* w, int32_t B, float* ranges, float* velocity, int32_t* hit, void* stream) {
  if (int rc = world_ready(w, B, "nb_world_scan", true)) return rc;
  if (!ranges) return fail(NB_ERR_INVALID, "nb_world_scan: null ranges");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  // the dynamic shared-memory limit is an attribute of the kernel, shared by every handle of the process: set this handle's
  // size before each launch (another handle's nb_world_set_scenes may have set a smaller one)
  auto* kernel = w->ep_slots ? (w->has_map ? nb::world_scan_kernel<true, true> : nb::world_scan_kernel<false, true>)
                             : (w->has_map ? nb::world_scan_kernel<true, false> : nb::world_scan_kernel<false, false>);
  NB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(w->scan_smem, 1)));
  kernel<<<w->scan_grid, w->scan_threads, w->scan_smem, (cudaStream_t)stream>>>(world_params(w), world_map_params(w), w->max_circ, w->max_edges,
                                                                                w->max_redges, ranges, velocity, hit);
  ++nb::launches;
  NB_CUDA(cudaGetLastError());
  return NB_OK;
}

int nb_world_step(nb_world_t* w, int32_t B, const float* action, int32_t* collided, int32_t* arrived, float* clearance, void* stream) {
  if (int rc = world_ready(w, B, "nb_world_step", true)) return rc;
  if (!action) return fail(NB_ERR_INVALID, "nb_world_step: null action");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  const nb::WorldParams prm = world_params(w);  // prm.B: the environments, or the slots in episode mode
  if (w->has_rvo) {  // reactive obstacles choose their velocities from the states at the start of the step
    const int grid = std::min(w->rvo_grid, prm.B);
    if (w->has_block) {
      auto* rvo = w->ep_slots ? nb::world_rvo_block_kernel<true> : nb::world_rvo_block_kernel<false>;
      NB_CUDA(cudaFuncSetAttribute(rvo, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)w->rvo_smem));
      rvo<<<grid, 32 * nb::kWorldRvoWarps, w->rvo_smem, (cudaStream_t)stream>>>(prm, world_rvo_params(w, action), world_map_params(w), world_block_params(w));
    } else {
      auto* rvo = w->ep_slots ? nb::world_rvo_kernel<true> : nb::world_rvo_kernel<false>;
      NB_CUDA(cudaFuncSetAttribute(rvo, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)w->rvo_smem));
      rvo<<<grid, 32 * nb::kWorldRvoWarps, w->rvo_smem, (cudaStream_t)stream>>>(prm, world_rvo_params(w, action));
    }
    ++nb::launches;
    NB_CUDA(cudaGetLastError());
  }
  // a CTA of up to 8 warps per E environments, a warp per robot
  const int E = nb::world_step_envs(w->K);
  const dim3 grid((prm.B + E - 1) / E), block(32 * std::min(E * w->K, nb::kWorldStepMaxWarps));
  if (w->has_block) {
    auto* kernel = w->ep_slots ? nb::world_step_block_kernel<true> : nb::world_step_block_kernel<false>;
    kernel<<<grid, block, 0, (cudaStream_t)stream>>>(prm, world_map_params(w), world_block_params(w), action, collided, arrived, clearance);
  } else {
    auto* kernel = w->ep_slots ? (w->has_map ? nb::world_step_ep_kernel<true> : nb::world_step_ep_kernel<false>)
                               : (w->has_map ? nb::world_step_kernel<true> : nb::world_step_kernel<false>);
    kernel<<<grid, block, 0, (cudaStream_t)stream>>>(prm, world_map_params(w), action, collided, arrived, clearance);
  }
  ++nb::launches;
  NB_CUDA(cudaGetLastError());
  if (w->ep_slots) {  // end the episodes of this step and hand out the next scenes
    nb::WorldEpisodeParams ep;
    ep.S = w->B; ep.slots = w->ep_slots; ep.K = w->K; ep.max_steps = w->ep_max_steps;
    ep.scene_of = w->d_scene_of; ep.live = w->d_live; ep.reset = w->d_reset; ep.t = w->d_ep_t;
    ep.next = w->d_ep_count; ep.finished = w->d_ep_count + 1;
    ep.collided = w->d_collided; ep.arrived = w->d_arrived; ep.clear = w->d_ep_clear;
    ep.r_col = w->d_r_col; ep.r_arr = w->d_r_arr; ep.r_astep = w->d_r_astep; ep.r_minclr = w->d_r_minclr;
    ep.r_end = w->d_r_end; ep.r_reason = w->d_r_reason; ep.r_slot = w->d_r_slot;
    nb::world_advance_kernel<<<1, nb::kWorldAdvanceThreads, 0, (cudaStream_t)stream>>>(ep);
    ++nb::launches;
    NB_CUDA(cudaGetLastError());
  }
  return NB_OK;
}

int nb_world_read_state(nb_world_t* w, int32_t B, double* states, double* obstacles, int32_t* collided, int32_t* arrived, void* stream) {
  // episode mode: B = slots K reads the slot rows (a gather), B = S K the scenes' own rows (copies, like a plain world)
  const bool scenes = w && w->ep_slots && B == w->B * w->K;
  if (!scenes)
    if (int rc = world_ready(w, B, "nb_world_read_state", true)) return rc;
  NB_CUDA(cudaSetDevice(w->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  if (w->ep_slots && !scenes) {
    if (obstacles && w->O) NB_CUDA(cudaMemcpyAsync(obstacles, w->d_obs, sizeof(double) * nb::kWorldObsCols * w->O, cudaMemcpyDeviceToDevice, st));
    if (!states && !collided && !arrived) return NB_OK;
    nb::world_gather_kernel<<<(B + 255) / 256, 256, 0, st>>>(w->ep_slots, w->K, w->d_scene_of, w->d_states, w->d_collided, w->d_arrived, states,
                                                             collided, arrived);
    ++nb::launches;
    NB_CUDA(cudaGetLastError());
    return NB_OK;
  }
  if (states) NB_CUDA(cudaMemcpyAsync(states, w->d_states, sizeof(double) * 3 * B, cudaMemcpyDeviceToDevice, st));
  if (obstacles && w->O) NB_CUDA(cudaMemcpyAsync(obstacles, w->d_obs, sizeof(double) * nb::kWorldObsCols * w->O, cudaMemcpyDeviceToDevice, st));
  if (collided) NB_CUDA(cudaMemcpyAsync(collided, w->d_collided, sizeof(int32_t) * B, cudaMemcpyDeviceToDevice, st));
  if (arrived) NB_CUDA(cudaMemcpyAsync(arrived, w->d_arrived, sizeof(int32_t) * B, cudaMemcpyDeviceToDevice, st));
  return NB_OK;
}

int nb_world_check_fleet_ex(const nb_world_config* cfg, int32_t T, const nb_world_robot_type* types, int32_t B, int32_t K, const double* robots,
                            const int32_t* robot_type) {
  return world_check_fleet(cfg, T, types, B, K, robots, robot_type);
}

int nb_world_check_fleet(const nb_world_config* cfg, int32_t B, int32_t K, const double* robots) {
  return nb_world_check_fleet_ex(cfg, 0, nullptr, B, K, robots, nullptr);
}

int nb_world_set_fleet_ex(nb_world_t* w, int32_t T, const nb_world_robot_type* types, int32_t B, int32_t K, const double* robots,
                          const int32_t* robot_type) {
  if (int rc = world_ready(w, B, "nb_world_set_fleet")) return rc;
  if (int rc = world_check_fleet(&w->cfg, T, types, B, K, robots, robot_type)) return rc;
  NB_CUDA(cudaSetDevice(w->cfg.device));
  w->B = 0;  // unusable until the new arrays are in place
  world_drop_maps(w);  // the new starts need a new map check
  world_drop_episodes(w);
  if (int rc = world_set_robots(w, B, K, robots, T, types, robot_type)) return rc;
  if (int rc = world_scan_shape(w, B)) return rc;
  if (w->d_beh)
    if (int rc = world_rvo_shape(w, B)) return rc;
  w->B = B;
  NB_CUDA(cudaDeviceSynchronize());
  return NB_OK;
}

int nb_world_set_fleet(nb_world_t* w, int32_t B, int32_t K, const double* robots) {
  return nb_world_set_fleet_ex(w, 0, nullptr, B, K, robots, nullptr);
}

int nb_world_check_maps(const nb_world_config* cfg, int32_t T, const nb_world_robot_type* types, int32_t B, int32_t K, const double* robots,
                        const int32_t* robot_type, int32_t P, const nb_world_map* maps, const uint32_t* bits, const int32_t* env_map,
                        double window) {
  return world_check_maps(cfg, T, types, B, K, robots, robot_type, P, maps, bits, env_map, window, nullptr);
}

int nb_world_set_maps(nb_world_t* w, int32_t P, const nb_world_map* maps, const uint32_t* bits, const int32_t* env_map, double window) {
  if (!w) return fail(NB_ERR_INVALID, "nb_world_set_maps: null handle");
  if (int rc = world_ready(w, w->B, "nb_world_set_maps")) return rc;
  std::vector<nb::WorldMap> table;
  if (int rc = world_check_maps(&w->cfg, (int32_t)w->h_types.size(), w->h_types.data(), w->B, w->K, w->h_robots.data(), w->h_rtype.data(), P, maps,
                                bits, env_map, window, &table))
    return rc;
  NB_CUDA(cudaSetDevice(w->cfg.device));
  world_drop_maps(w);
  world_drop_episodes(w);
  const size_t words = (size_t)(table.back().off + (int64_t)table.back().H * table.back().words);
  cudaError_t e = nb::dalloc(&w->d_maps, table.size());
  if (e == cudaSuccess) e = nb::dalloc(&w->d_bits, words);
  if (e == cudaSuccess) e = nb::dalloc(&w->d_env_map, (size_t)w->B);
  if (e == cudaSuccess) e = cudaMemcpy(w->d_maps, table.data(), sizeof(nb::WorldMap) * table.size(), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(w->d_bits, bits, sizeof(uint32_t) * words, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(w->d_env_map, env_map, sizeof(int32_t) * w->B, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {  // the handle stays usable, without maps
    cudaGetLastError();
    world_drop_maps(w);
    if (int rc = world_scan_shape(w, w->B)) return rc;
    return fail(NB_ERR_CUDA, "nb_world_set_maps: %zu words of maps: %s", words, cudaGetErrorString(e));
  }
  w->has_map = std::any_of(env_map, env_map + w->B, [](int32_t m) { return m >= 0; });
  w->window = window;
  w->h_maps = table;
  w->h_bits.assign(bits, bits + words);
  w->h_env_map.assign(env_map, env_map + w->B);
  if (int rc = world_scan_shape(w, w->B)) return rc;
  NB_CUDA(cudaDeviceSynchronize());
  return NB_OK;
}

int nb_world_check_episodes(const nb_world_config* cfg, int32_t S, int32_t K, const int32_t* robot_type, int32_t slots, int32_t max_steps) {
  return world_check_episodes(cfg, S, K, robot_type, slots, max_steps);
}

int nb_world_set_episodes(nb_world_t* w, int32_t slots, int32_t max_steps) {
  if (!w) return fail(NB_ERR_INVALID, "nb_world_set_episodes: null handle");
  if (int rc = world_ready(w, w->B, "nb_world_set_episodes")) return rc;
  const int S = w->B, K = w->K;
  if (int rc = world_check_episodes(&w->cfg, S, K, w->h_rtype.data(), slots, max_steps)) return rc;
  NB_CUDA(cudaSetDevice(w->cfg.device));
  world_drop_episodes(w);
  const size_t SK = (size_t)S * K, BK = (size_t)slots * K;
  std::vector<int32_t> scene_of(slots), slot(S, -1), minus(SK, -1);
  for (int b = 0; b < slots; ++b) scene_of[b] = slot[b] = b;
  const int32_t count[2] = {slots, 0};  // the next scene, episodes finished
  std::vector<float> inf(SK, INFINITY);
  cudaError_t e = cudaSuccess;
  auto alloc = [&](auto** p, size_t n) { if (e == cudaSuccess) e = dalloc(p, std::max<size_t>(n, 1)); };
  alloc(&w->d_scene_of, slots); alloc(&w->d_live, slots); alloc(&w->d_reset, slots); alloc(&w->d_ep_t, slots); alloc(&w->d_ep_count, 2);
  alloc(&w->d_ep_clear, BK);
  alloc(&w->d_r_col, SK); alloc(&w->d_r_arr, SK); alloc(&w->d_r_astep, SK); alloc(&w->d_r_minclr, SK);
  alloc(&w->d_r_end, S); alloc(&w->d_r_reason, S); alloc(&w->d_r_slot, S);
  auto up = [&](void* d, const void* h, size_t bytes) { if (e == cudaSuccess) e = cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice); };
  auto one = [&](void* d, size_t n) {  // int32 ones
    std::vector<int32_t> v(n, 1);
    up(d, v.data(), n * sizeof(int32_t));
  };
  up(w->d_scene_of, scene_of.data(), slots * sizeof(int32_t));
  one(w->d_live, slots);
  one(w->d_reset, slots);  // every slot has just taken its first scene
  if (e == cudaSuccess) e = cudaMemset(w->d_ep_t, 0, slots * sizeof(int32_t));
  up(w->d_ep_count, count, sizeof(count));
  if (e == cudaSuccess) e = cudaMemset(w->d_r_col, 0, SK * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMemset(w->d_r_arr, 0, SK * sizeof(int32_t));
  up(w->d_r_astep, minus.data(), SK * sizeof(int32_t));
  up(w->d_r_minclr, inf.data(), SK * sizeof(float));
  if (e == cudaSuccess) e = cudaMemset(w->d_r_end, 0, S * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMemset(w->d_r_reason, 0, S * sizeof(int32_t));
  up(w->d_r_slot, slot.data(), S * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {  // the handle stays usable as a plain world
    cudaGetLastError();
    world_drop_episodes(w);
    return fail(NB_ERR_CUDA, "nb_world_set_episodes: %s", cudaGetErrorString(e));
  }
  w->ep_slots = slots; w->ep_max_steps = max_steps;
  return NB_OK;
}

int nb_world_read_episodes(nb_world_t* w, int32_t S, int32_t* collided, int32_t* arrived, int32_t* arrive_step, float* min_clearance, int32_t* end_step,
                           int32_t* reason, int32_t* slot, int32_t* scene_of, int32_t* reset, int32_t* finished, void* stream) {
  if (int rc = world_ready(w, S, "nb_world_read_episodes")) return rc;
  if (!w->ep_slots) return fail(NB_ERR_INVALID, "nb_world_read_episodes: not in episode mode (nb_world_set_episodes)");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t SK = (size_t)S * w->K;
  auto cp = [&](void* dst, const void* src, size_t bytes) { return dst ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st) : cudaSuccess; };
  NB_CUDA(cp(collided, w->d_r_col, SK * sizeof(int32_t)));
  NB_CUDA(cp(arrived, w->d_r_arr, SK * sizeof(int32_t)));
  NB_CUDA(cp(arrive_step, w->d_r_astep, SK * sizeof(int32_t)));
  NB_CUDA(cp(min_clearance, w->d_r_minclr, SK * sizeof(float)));
  NB_CUDA(cp(end_step, w->d_r_end, S * sizeof(int32_t)));
  NB_CUDA(cp(reason, w->d_r_reason, S * sizeof(int32_t)));
  NB_CUDA(cp(slot, w->d_r_slot, S * sizeof(int32_t)));
  NB_CUDA(cp(scene_of, w->d_scene_of, w->ep_slots * sizeof(int32_t)));
  NB_CUDA(cp(reset, w->d_reset, w->ep_slots * sizeof(int32_t)));
  NB_CUDA(cp(finished, w->d_ep_count + 1, sizeof(int32_t)));
  return NB_OK;
}

int nb_world_check_map_contact(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obstacles, const int32_t* vert_begin,
                               const double* vertices, const double* envs, const int32_t* obs_kind, const double* behaviors, int32_t P,
                               const nb_world_map* maps, const uint32_t* bits, const int32_t* env_map, const int32_t* flags) {
  if (int rc = world_check_scenes(cfg, B, obs_begin, obstacles, vert_begin, vertices, envs, obs_kind, nullptr, nullptr, nullptr, nullptr)) return rc;
  if (behaviors)
    if (int rc = world_check_behaviors(cfg, B, obs_begin, obstacles, envs, behaviors)) return rc;
  std::vector<nb::WorldMap> table;
  if (int rc = world_check_maps(cfg, 0, nullptr, B, 1, nullptr, nullptr, P, maps, bits, env_map, 1.0, &table)) return rc;
  return world_check_contact(cfg, B, obs_begin, obstacles, vert_begin, vertices, obs_kind, behaviors, table, bits, env_map, flags);
}

int nb_world_set_map_contact(nb_world_t* w, int32_t B, const int32_t* flags) {
  if (int rc = world_ready(w, B, "nb_world_set_map_contact")) return rc;
  if (!w->d_maps) return fail(NB_ERR_INVALID, "nb_world_set_map_contact: no maps set (nb_world_set_maps)");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  const int O = w->O;
  std::vector<double> obs((size_t)nb::kWorldObsCols * O), beh;
  if (O) NB_CUDA(cudaMemcpy(obs.data(), w->d_obs, sizeof(double) * obs.size(), cudaMemcpyDeviceToHost));  // the current centres
  if (w->d_beh && O) {
    beh.resize((size_t)nb::kWorldBehCols * O);
    NB_CUDA(cudaMemcpy(beh.data(), w->d_beh, sizeof(double) * beh.size(), cudaMemcpyDeviceToHost));
  }
  if (int rc = world_check_contact(&w->cfg, B, w->h_obs_begin.data(), obs.data(), w->h_vert_begin.data(), w->h_vertices.data(), w->h_kind.data(),
                                   beh.empty() ? nullptr : beh.data(), w->h_maps, w->h_bits.data(), w->h_env_map.data(), flags))
    return rc;
  world_drop_contact(w);
  world_drop_episodes(w);
  // a wandering obstacle without an explicit goal in a blocking environment starts from goal = its centre and draw 0, so that its
  // first goal is drawn on the device through the map test
  std::vector<double> goal;
  std::vector<int32_t> draws;
  bool reset = false;
  if (!beh.empty()) {
    goal.resize(2 * (size_t)O); draws.resize(O);
    NB_CUDA(cudaMemcpy(goal.data(), w->d_goal, sizeof(double) * goal.size(), cudaMemcpyDeviceToHost));
    NB_CUDA(cudaMemcpy(draws.data(), w->d_draws, sizeof(int32_t) * O, cudaMemcpyDeviceToHost));
    for (int b = 0; b < B; ++b) {
      if (!flags[b]) continue;
      for (int o = w->h_obs_begin[b]; o < w->h_obs_begin[b + 1]; ++o) {
        const double* r = beh.data() + (size_t)nb::kWorldBehCols * o;
        if (r[0] != 1.0 || r[6] == 0.0 || !std::isnan(r[7])) continue;
        goal[2 * o] = obs[(size_t)nb::kWorldObsCols * o]; goal[2 * o + 1] = obs[(size_t)nb::kWorldObsCols * o + 1];
        draws[o] = 0;
        reset = true;
      }
    }
  }
  cudaError_t e = nb::dalloc(&w->d_block, (size_t)B);
  if (e == cudaSuccess) e = nb::dalloc(&w->d_bounces, std::max<size_t>(O, 1));
  if (e == cudaSuccess) e = nb::dalloc(&w->d_bounced, std::max<size_t>(O, 1));
  if (e == cudaSuccess) e = cudaMemcpy(w->d_block, flags, sizeof(int32_t) * B, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemset(w->d_bounces, 0, sizeof(int32_t) * std::max(O, 1));
  if (e == cudaSuccess) e = cudaMemset(w->d_bounced, 0, sizeof(int32_t) * std::max(O, 1));
  if (e == cudaSuccess && reset) e = cudaMemcpy(w->d_goal, goal.data(), sizeof(double) * goal.size(), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && reset) e = cudaMemcpy(w->d_draws, draws.data(), sizeof(int32_t) * O, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    cudaGetLastError();
    world_drop_contact(w);
    return fail(NB_ERR_CUDA, "nb_world_set_map_contact: %s", cudaGetErrorString(e));
  }
  w->has_block = std::any_of(flags, flags + B, [](int32_t f) { return f != 0; });
  return NB_OK;
}

int nb_world_read_map_contact(nb_world_t* w, int32_t O, int32_t* bounces, void* stream) {
  if (!w) return fail(NB_ERR_INVALID, "nb_world_read_map_contact: null handle");
  if (!w->d_bounces) return fail(NB_ERR_INVALID, "nb_world_read_map_contact: no map contact set (nb_world_set_map_contact)");
  if (O != w->O) return fail(NB_ERR_INVALID, "nb_world_read_map_contact: O = %d but the scenes have %d obstacles", O, w->O);
  if (!bounces) return fail(NB_ERR_INVALID, "nb_world_read_map_contact: null bounces");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  if (O) NB_CUDA(cudaMemcpyAsync(bounces, w->d_bounces, sizeof(int32_t) * O, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return NB_OK;
}

}  // extern "C"
