// C ABI of the batched 2-D world (nb_world_*, include/neupan_b200.h): the host-side checks of configs, scenes, behaviours and fleets,
// the world handle, and the launches of the scan, rvo and step kernels.
#include <algorithm>
#include <cmath>
#include <memory>
#include <new>
#include <vector>

#include "host_common.h"
#include "world_kernel.cuh"
#include "world_rvo_kernel.cuh"
#include "world_episode_kernel.cuh"
#include "world_contact_kernel.cuh"

using nb::fail;

struct nb_world {
  nb_world_config cfg;
  int B = 0, O = 0, V = 0;
  int max_circ = 0, max_edges = 0, scan_threads = 0, scan_grid = 0;
  size_t scan_smem = 0;
  nb::DeviceArray<double> beam_cs;  // (R, 2), fixed at creation
  // the scenes (nb_world_set_scenes_ex)
  struct Scenes {
    nb::DeviceArray<int32_t> obs_begin, vert_begin, slot, counts, kind;
    nb::DeviceArray<double> vertices, env, obs;
  } scenes;
  // host copies of the scene (nb_world_set_behaviors checks against them)
  std::vector<int32_t> h_obs_begin, h_vert_begin, h_kind;
  std::vector<double> h_vertices, h_env;
  // obstacle behaviours (nb_world_set_behaviors): has_rvo false -> nb_world_step launches only world_step_kernel
  struct Behaviors {
    bool has_rvo = false;
    uint64_t seed = 0;
    int cap = 0, grid = 0;
    size_t smem = 0;
    int max_n = 0;  // the largest environment's obstacle count (cap = max_n + K)
    nb::DeviceArray<double> beh, rad, goal;
    nb::DeviceArray<int32_t> draws;
  } rvo;
  // robots per environment (nb_world_set_fleet; nb_world_set_scenes makes it 1, from the env rows): the per-robot arrays hold B K
  // rows (world_set_robots): states, flags, every robot's goal and the velocity of its last step; the robot types (type 0 is the
  // config's robot): the table (T + 1 rows) and each robot's type (B K, zeros without a mix)
  int K = 1;
  struct Robots {
    nb::DeviceArray<double> states, goal, vel, cmd;  // cmd: cmd_prev (B K, 2), the last limited command (nb_world_set_actuation)
    nb::DeviceArray<int32_t> collided, arrived, rtype;
    nb::DeviceArray<nb::WorldRobotType> types;
  } robots;
  int max_redges = 0;  // the largest environment's robot edge count (the scan's staging size; 0 with K = 1)
  // host copies of the placed robots (nb_world_set_maps checks the start bodies against them): rows, types 1..T, each robot's type
  std::vector<double> h_robots;
  std::vector<nb_world_robot_type> h_types;
  std::vector<int32_t> h_rtype;
  // occupancy maps (nb_world_set_maps): has_map false -> the kernels' map-free instantiations; the host copies are what
  // nb_world_set_map_contact checks the obstacles' starts against
  struct Maps {
    bool has_map = false;
    nb::DeviceArray<nb::WorldMap> table;
    nb::DeviceArray<uint32_t> bits;
    nb::DeviceArray<int32_t> env_map;
    double window = 0.0;
    std::vector<nb::WorldMap> h_table;
    std::vector<uint32_t> h_bits;
    std::vector<int32_t> h_env_map;
  } maps;
  // maps that block obstacles (nb_world_set_map_contact): has_block false -> the kernels' instantiations without it
  struct Contact {
    bool has_block = false;
    nb::DeviceArray<int32_t> block, bounces, bounced;
  } contact;
  // obstacles that block each other (nb_world_set_obstacle_contact): has_contact false -> the kernels of a world without it
  struct ObstacleContact {
    bool has_contact = false;
    int max_n = 0;  // the largest environment's obstacle count (world_contact_kernel's staging)
    nb::DeviceArray<int32_t> flag, bounces;
  } ocontact;
  // episode mode (nb_world_set_episodes): slots > 0 slots run the B = S scenes of the bank
  struct Episodes {
    int slots = 0, max_steps = 0;
    nb::DeviceArray<int32_t> scene_of, live, reset, t, count;  // count: next, finished
    nb::DeviceArray<float> clear;
    nb::DeviceArray<int32_t> r_col, r_arr, r_astep, r_end, r_reason, r_slot;
    nb::DeviceArray<float> r_minclr;
  } ep;
  // actuation limits and motion noise (nb_world_set_actuation): on false -> the step kernels without the actuation stage; act holds
  // kWorldMaxRobotTypes rows (defaults past num_types).  Kept by nb_world_set_scenes / _fleet / _episodes, which zero cmd_prev.
  struct Actuation {
    bool on = false;
    uint64_t seed = 0;
    nb::DeviceArray<double> act;
  } act;
  // lidar range noise (nb_world_set_lidar_noise): range_std 0 -> the scan kernels without it
  double range_min = 0.0, range_std = 0.0;
  uint64_t lidar_seed = 0;
  uint64_t steps = 0;  // plain world: nb_world_step calls since the robots were placed (the noise streams' step n)
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

// ---- obstacle contact on the host (the start check of nb_world_set_obstacle_contact) ------------------------------------------

double host_seg_dist(double px, double py, const double* a, const double* b) {
  const double ex = b[0] - a[0], ey = b[1] - a[1], wx = px - a[0], wy = py - a[1];
  double t = (host_dmul(wx, ex) + host_dmul(wy, ey)) / (host_dmul(ex, ex) + host_dmul(ey, ey));
  t = t < 0.0 ? 0.0 : (t > 1.0 ? 1.0 : t);
  const double qx = wx - host_dmul(t, ex), qy = wy - host_dmul(t, ey);
  return std::sqrt(host_dmul(qx, qx) + host_dmul(qy, qy));
}

double host_cross(const double* a, const double* b, double px, double py) {
  return host_dmul(b[0] - a[0], py - a[1]) - host_dmul(b[1] - a[1], px - a[0]);
}

// even-odd test of (px, py) against the polygon v of n vertices
bool host_inside_outline(const double* v, int n, double px, double py) {
  bool in = false;
  for (int k = 0; k < n; ++k) {
    const double* a = v + 2 * k;
    const double* b = v + 2 * ((k + 1) % n);
    if ((a[1] > py) != (b[1] > py)) {
      const double cr = host_cross(a, b, px, py);
      if (b[1] > a[1] ? cr > 0.0 : cr < 0.0) in = !in;
    }
  }
  return in;
}

// (px, py) is not strictly outside the convex polygon v (the edge cross products do not take both signs)
bool host_inside_convex(const double* v, int n, double px, double py) {
  bool pos = false, neg = false;
  for (int k = 0; k < n; ++k) {
    const double cr = host_cross(v + 2 * k, v + 2 * ((k + 1) % n), px, py);
    pos |= cr > 0.0; neg |= cr < 0.0;
  }
  return !(pos && neg);
}

// An obstacle footprint at its centre: rank 0 circle, 1 convex polygon, 2 outline; world vertices; the box widened by the pad
struct HostShape {
  double cx, cy, r;
  int nv, rank;
  double v[2 * nb::kWorldMaxOutlineVertices];
  double box[4];
};

HostShape host_shape(const double* row, const double* rel, int nv, int kind) {
  HostShape s{};
  s.cx = row[0]; s.cy = row[1]; s.r = row[4]; s.nv = nv;
  s.rank = nv == 0 ? 0 : (kind != 0 ? 2 : 1);
  double x0 = -s.r, y0 = -s.r, x1 = s.r, y1 = s.r;
  if (nv > 0) {
    x0 = x1 = rel[0]; y0 = y1 = rel[1];
    for (int k = 0; k < nv; ++k) {
      s.v[2 * k] = s.cx + rel[2 * k]; s.v[2 * k + 1] = s.cy + rel[2 * k + 1];
      x0 = std::min(x0, rel[2 * k]); x1 = std::max(x1, rel[2 * k]);
      y0 = std::min(y0, rel[2 * k + 1]); y1 = std::max(y1, rel[2 * k + 1]);
    }
  }
  s.box[0] = s.cx + x0 - nb::kWorldContactPad; s.box[1] = s.cy + y0 - nb::kWorldContactPad;
  s.box[2] = s.cx + x1 + nb::kWorldContactPad; s.box[3] = s.cy + y1 + nb::kWorldContactPad;
  return s;
}

// world_footprints_touch on the host, behind the same broad phase
bool host_shapes_touch(const HostShape& f, const HostShape& g) {
  if (f.box[2] < g.box[0] || g.box[2] < f.box[0] || f.box[3] < g.box[1] || g.box[3] < f.box[1]) return false;
  const HostShape& a = f.rank <= g.rank ? f : g;
  const HostShape& b = f.rank <= g.rank ? g : f;
  if (b.rank == 0) {
    const double dx = a.cx - b.cx, dy = a.cy - b.cy;
    return std::sqrt(host_dmul(dx, dx) + host_dmul(dy, dy)) - (a.r + b.r) <= 0.0;
  }
  if (a.rank == 0) {
    double d = INFINITY;
    for (int k = 0; k < b.nv; ++k) d = std::min(d, host_seg_dist(a.cx, a.cy, b.v + 2 * k, b.v + 2 * ((k + 1) % b.nv)));
    return b.rank == 1 ? (host_inside_convex(b.v, b.nv, a.cx, a.cy) || d - a.r <= 0.0) : (host_inside_outline(b.v, b.nv, a.cx, a.cy) || d <= a.r);
  }
  if (b.rank == 1) return world_bodies_meet(a.v, a.nv, b.v, b.nv);
  for (int k = 0; k < a.nv; ++k)
    for (int i = 0; i < b.nv; ++i)
      if (world_segs_meet(a.v + 2 * k, a.v + 2 * ((k + 1) % a.nv), b.v + 2 * i, b.v + 2 * ((i + 1) % b.nv))) return true;
  if (host_inside_outline(b.v, b.nv, a.v[0], a.v[1])) return true;
  return a.rank == 1 ? host_inside_convex(a.v, a.nv, b.v[0], b.v[1]) : host_inside_outline(a.v, a.nv, b.v[0], b.v[1]);
}

// Every check of nb_world_set_obstacle_contact on valid scenes and behaviours (NULL: every obstacle constant); obs holds the
// obstacles' current centres and velocities.
int world_check_obstacle_contact(int32_t B, const int32_t* obs_begin, const double* obs, const int32_t* vert_begin, const double* vertices,
                                 const int32_t* kind, const double* beh, const int32_t* flags) {
  if (!flags) return fail(NB_ERR_INVALID, "nb_world obstacle contact: null flags");
  std::vector<HostShape> shapes;
  for (int b = 0; b < B; ++b) {
    if (flags[b] != 0 && flags[b] != 1) return fail(NB_ERR_INVALID, "environment %d: obstacle contact flag %d (0 or 1)", b, flags[b]);
    if (flags[b] == 0) continue;
    const int o0 = obs_begin[b], o1 = obs_begin[b + 1];
    shapes.clear();
    for (int o = o0; o < o1; ++o)
      shapes.push_back(host_shape(obs + (size_t)nb::kWorldObsCols * o, vertices + 2 * (size_t)vert_begin[o], vert_begin[o + 1] - vert_begin[o],
                                  kind ? kind[o] : 0));
    for (int o = o0; o < o1; ++o) {
      const double* row = obs + (size_t)nb::kWorldObsCols * o;
      const bool reactive = beh && beh[(size_t)nb::kWorldBehCols * o] == 1.0;
      if (!reactive && row[2] == 0.0 && row[3] == 0.0) continue;  // static obstacles may overlap each other
      for (int p = o0; p < o1; ++p)
        if (p != o && host_shapes_touch(shapes[o - o0], shapes[p - o0]))
          return fail(NB_ERR_INVALID, "environment %d, obstacle %d: moves but its start footprint overlaps or touches obstacle %d", b, o, p);
    }
  }
  return NB_OK;
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

nb::WorldMapParams world_map_params(const nb_world* w) {
  return nb::WorldMapParams{w->maps.table.get(), w->maps.bits.get(), w->maps.env_map.get(), w->maps.window};
}
nb::WorldBlockParams world_block_params(const nb_world* w) {
  return nb::WorldBlockParams{w->contact.block.get(), w->contact.bounces.get(), w->contact.bounced.get()};
}
nb::WorldContactParams world_contact_params(const nb_world* w) {
  return nb::WorldContactParams{w->ocontact.flag.get(), w->ocontact.bounces.get(), w->ocontact.max_n};
}

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
  if (int rc = w->maps.has_map ? world_scan_occupancy<true>(w, &per_sm) : world_scan_occupancy<false>(w, &per_sm)) return rc;
  NB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, w->cfg.device));
  if (per_sm < 1) return fail(NB_ERR_CUDA, "world_scan_kernel: %zu B of shared memory do not fit", w->scan_smem);
  w->scan_grid = std::min(B, per_sm * sms);
  return NB_OK;
}

// rvo launch shape: the largest environment's rows (+ the K robots) and one cone list per warp in shared memory
int world_rvo_shape(nb_world* w, int B) {
  nb_world::Behaviors& r = w->rvo;
  r.cap = r.max_n + w->K;
  r.smem = (size_t)r.cap * (5 * sizeof(double) + nb::kWorldRvoWarps * (6 * sizeof(double) + sizeof(int32_t)));
  NB_CUDA(cudaFuncSetAttribute(nb::world_rvo_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)r.smem));
  int per_sm = 0, sms = 0;
  NB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, nb::world_rvo_kernel<false>, 32 * nb::kWorldRvoWarps, r.smem));
  NB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, w->cfg.device));
  if (per_sm < 1) return fail(NB_ERR_CUDA, "world_rvo_kernel: %zu B of shared memory do not fit", r.smem);
  r.grid = std::min(B, per_sm * sms);
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
  nb_world::Robots& r = w->robots;
  r = {};
  NB_CUDA(nb::alloc(r.states, 3 * N));
  NB_CUDA(nb::alloc(r.collided, N));
  NB_CUDA(nb::alloc(r.arrived, N));
  NB_CUDA(nb::alloc(r.goal, 3 * N));
  NB_CUDA(nb::alloc(r.vel, 2 * N));
  NB_CUDA(nb::alloc(r.cmd, 2 * N));
  NB_CUDA(nb::alloc(r.types, table.size()));
  NB_CUDA(nb::alloc(r.rtype, N));
  NB_CUDA(cudaMemcpy(r.states.get(), states.data(), sizeof(double) * 3 * N, cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(r.goal.get(), goal.data(), sizeof(double) * 3 * N, cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(r.types.get(), table.data(), sizeof(nb::WorldRobotType) * table.size(), cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(r.rtype.get(), rtype.data(), sizeof(int32_t) * N, cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemset(r.collided.get(), 0, sizeof(int32_t) * N));
  NB_CUDA(cudaMemset(r.arrived.get(), 0, sizeof(int32_t) * N));
  NB_CUDA(cudaMemset(r.vel.get(), 0, sizeof(double) * 2 * N));
  NB_CUDA(cudaMemset(r.cmd.get(), 0, sizeof(double) * 2 * N));
  w->K = K;
  w->steps = 0;
  w->max_redges = max_redges;
  w->h_robots.assign(robots, robots + 6 * N);
  w->h_types.assign(types, types + T);
  w->h_rtype = rtype;
  return NB_OK;
}

nb::WorldParams world_params(const nb_world* w) {
  nb::WorldParams prm;
  const nb_world_config& c = w->cfg;
  const nb_world::Scenes& s = w->scenes;
  const nb_world::Robots& r = w->robots;
  prm.B = w->ep.slots ? w->ep.slots : w->B; prm.R = c.num_beams;
  prm.dt = c.step_time; prm.range_max = c.range_max; prm.beam_cs = w->beam_cs.get();
  prm.off_x = c.scan_offset[0]; prm.off_y = c.scan_offset[1]; prm.off_th = c.scan_offset[2];
  prm.types = r.types.get(); prm.rtype = r.rtype.get();
  prm.obs_begin = s.obs_begin.get(); prm.vert_begin = s.vert_begin.get(); prm.slot = s.slot.get(); prm.counts = s.counts.get(); prm.kind = s.kind.get();
  prm.vertices = s.vertices.get(); prm.env = s.env.get(); prm.obs = s.obs.get(); prm.states = r.states.get();
  prm.collided = r.collided.get(); prm.arrived = r.arrived.get();
  prm.K = w->K; prm.fgoal = r.goal.get(); prm.fvel = r.vel.get();
  prm.scene_of = w->ep.scene_of.get(); prm.live = w->ep.live.get(); prm.ep_clear = w->ep.clear.get();
  return prm;
}

// per_robot: the count argument is the robot count N = B K (B itself with one robot per environment), in episode mode the slot
// robots slots K; otherwise (the obstacle-side calls) the environment count B (S in episode mode)
int world_ready(const nb_world* w, int32_t B, const char* what, bool per_robot = false) {
  if (!w) return fail(NB_ERR_INVALID, "%s: null handle", what);
  if (!w->B) return fail(NB_ERR_INVALID, "%s: no scenes set (nb_world_set_scenes)", what);
  if (per_robot && w->ep.slots) {
    if (B != w->ep.slots * w->K)
      return fail(NB_ERR_INVALID, "%s: count = %d but the world runs episodes in %d slots x %d robots (N = %d)", what, B, w->ep.slots, w->K,
                  w->ep.slots * w->K);
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
  rp.beh = w->rvo.beh.get(); rp.radius = w->rvo.rad.get(); rp.goal = w->rvo.goal.get(); rp.draws = w->rvo.draws.get(); rp.action = action;
  rp.seed = w->rvo.seed; rp.cap = w->rvo.cap;
  return rp;
}

// the actuation (step) or lidar (scan) noise parameters
nb::WorldNoiseParams world_noise_params(const nb_world* w, bool lidar) {
  nb::WorldNoiseParams nz;
  nz.act = w->act.act.get(); nz.cmd = w->robots.cmd.get(); nz.ep_t = w->ep.t.get(); nz.n = w->steps;
  nz.seed = lidar ? w->lidar_seed : w->act.seed;
  nz.range_min = w->range_min; nz.range_std = w->range_std;
  return nz;
}

// Every check of nb_world_set_actuation: one row per robot type of the handle, no NaN, vel_min <= vel_max with vel_min < +inf and
// vel_max > -inf, acce > 0 (+inf: no rate limit), finite alpha >= 0, and an acker type's finite steering limits in (-pi/2, pi/2).
int world_check_actuation(const nb_world* w, int32_t num_types, const nb_world_actuation* per_type) {
  const int T = 1 + (int)w->h_types.size();
  if (num_types != T) return fail(NB_ERR_INVALID, "nb_world_set_actuation: num_types = %d but the handle has %d robot types", num_types, T);
  if (!per_type) return fail(NB_ERR_INVALID, "nb_world_set_actuation: null per_type");
  for (int t = 0; t < T; ++t) {
    const nb_world_actuation& a = per_type[t];
    const int kin = t == 0 ? w->cfg.kinematics : w->h_types[t - 1].kinematics;
    for (int j = 0; j < 2; ++j) {
      if (std::isnan(a.vel_min[j]) || std::isnan(a.vel_max[j]) || std::isnan(a.acce[j]))
        return fail(NB_ERR_INVALID, "nb_world_set_actuation: type %d, component %d: NaN limit", t, j);
      if (!(a.vel_min[j] <= a.vel_max[j]) || a.vel_min[j] == INFINITY || a.vel_max[j] == -INFINITY)
        return fail(NB_ERR_INVALID, "nb_world_set_actuation: type %d, component %d: vel_min = %g, vel_max = %g (need vel_min <= vel_max, "
                    "vel_min < inf, vel_max > -inf)", t, j, a.vel_min[j], a.vel_max[j]);
      if (!(a.acce[j] > 0.0)) return fail(NB_ERR_INVALID, "nb_world_set_actuation: type %d, component %d: acce = %g must be > 0", t, j, a.acce[j]);
    }
    for (int j = 0; j < 4; ++j)
      if (!std::isfinite(a.alpha[j]) || a.alpha[j] < 0.0)
        return fail(NB_ERR_INVALID, "nb_world_set_actuation: type %d: alpha[%d] = %g must be finite and >= 0", t, j, a.alpha[j]);
    const double h = 1.5707963267948966;
    if (kin == NB_KIN_ACKER)
      for (const double s : {a.vel_min[1], a.vel_max[1]})
        if (std::isfinite(s) && !(-h < s && s < h))
          return fail(NB_ERR_INVALID, "nb_world_set_actuation: type %d (acker): steering limit %g outside (-pi/2, pi/2)", t, s);
  }
  return NB_OK;
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
  std::unique_ptr<nb_world> w(new (std::nothrow) nb_world());
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
  NB_CUDA(nb::alloc(w->beam_cs, cs.size()));
  NB_CUDA(cudaMemcpy(w->beam_cs.get(), cs.data(), sizeof(double) * cs.size(), cudaMemcpyHostToDevice));
  *out = w.release();
  return NB_OK;
}

int nb_world_destroy(nb_world_t* w) {
  if (!w) return NB_OK;
  cudaSetDevice(w->cfg.device);
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
  w->B = 0;
  // new scenes: every obstacle keeps a constant velocity until nb_world_set_behaviors, has no map until nb_world_set_maps, and the
  // world runs as a plain world until nb_world_set_episodes
  w->scenes = {}; w->rvo = {}; w->maps = {}; w->contact = {}; w->ocontact = {}; w->ep = {};
  w->h_obs_begin.assign(obs_begin, obs_begin + B + 1);
  w->h_vert_begin.assign(vert_begin, vert_begin + O + 1);
  w->h_vertices.assign(vertices, vertices + 2 * (size_t)V);
  if (obs_kind) w->h_kind.assign(obs_kind, obs_kind + O);
  else w->h_kind.assign(O, 0);
  w->h_env.assign(envs, envs + (size_t)nb::kWorldEnvCols * B);
  nb_world::Scenes& s = w->scenes;
  NB_CUDA(nb::alloc(s.obs_begin, (size_t)B + 1));
  NB_CUDA(nb::alloc(s.vert_begin, (size_t)O + 1));
  NB_CUDA(nb::alloc(s.slot, (size_t)O));
  NB_CUDA(nb::alloc(s.counts, 2 * (size_t)B));
  NB_CUDA(nb::alloc(s.kind, (size_t)O));
  if (O && obs_kind) NB_CUDA(cudaMemcpy(s.kind.get(), obs_kind, sizeof(int32_t) * O, cudaMemcpyHostToDevice));
  else if (O) NB_CUDA(cudaMemset(s.kind.get(), 0, sizeof(int32_t) * O));
  NB_CUDA(nb::alloc(s.vertices, 2 * (size_t)V));
  NB_CUDA(nb::alloc(s.env, (size_t)nb::kWorldEnvCols * B));
  NB_CUDA(nb::alloc(s.obs, (size_t)nb::kWorldObsCols * O));
  NB_CUDA(cudaMemcpy(s.obs_begin.get(), obs_begin, sizeof(int32_t) * (B + 1), cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(s.vert_begin.get(), vert_begin, sizeof(int32_t) * (O + 1), cudaMemcpyHostToDevice));
  if (O) NB_CUDA(cudaMemcpy(s.slot.get(), slot.data(), sizeof(int32_t) * O, cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(s.counts.get(), counts.data(), sizeof(int32_t) * 2 * B, cudaMemcpyHostToDevice));
  if (V) NB_CUDA(cudaMemcpy(s.vertices.get(), vertices, sizeof(double) * 2 * V, cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(s.env.get(), envs, sizeof(double) * nb::kWorldEnvCols * B, cudaMemcpyHostToDevice));
  if (O) NB_CUDA(cudaMemcpy(s.obs.get(), obstacles, sizeof(double) * nb::kWorldObsCols * O, cudaMemcpyHostToDevice));
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
  if (O) NB_CUDA(cudaMemcpy(obs.data(), w->scenes.obs.get(), sizeof(double) * obs.size(), cudaMemcpyDeviceToHost));  // the current centres
  if (int rc = world_check_behaviors(&w->cfg, B, w->h_obs_begin.data(), obs.data(), w->h_env.data(), behaviors)) return rc;
  w->contact = {}; w->ocontact = {}; w->ep = {};  // which obstacles move has changed: the contact flags need their checks again
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
  nb_world::Behaviors& r = w->rvo;
  r = {};
  NB_CUDA(nb::alloc(r.beh, (size_t)nb::kWorldBehCols * O));
  NB_CUDA(nb::alloc(r.rad, (size_t)O));
  NB_CUDA(nb::alloc(r.goal, 2 * (size_t)O));
  NB_CUDA(nb::alloc(r.draws, (size_t)O));
  if (O) {
    NB_CUDA(cudaMemcpy(r.beh.get(), behaviors, sizeof(double) * nb::kWorldBehCols * O, cudaMemcpyHostToDevice));
    NB_CUDA(cudaMemcpy(r.rad.get(), rad.data(), sizeof(double) * O, cudaMemcpyHostToDevice));
    NB_CUDA(cudaMemcpy(r.goal.get(), goal.data(), sizeof(double) * 2 * O, cudaMemcpyHostToDevice));
    NB_CUDA(cudaMemcpy(r.draws.get(), draws.data(), sizeof(int32_t) * O, cudaMemcpyHostToDevice));
  }
  r.seed = seed;
  r.max_n = max_n;
  if (int rc = world_rvo_shape(w, B)) return rc;
  r.has_rvo = any;
  NB_CUDA(cudaDeviceSynchronize());
  return NB_OK;
}

int nb_world_read_behaviors(nb_world_t* w, int32_t B, double* goals, int32_t* draws, void* stream) {
  if (int rc = world_ready(w, B, "nb_world_read_behaviors")) return rc;
  if (!w->rvo.goal) return fail(NB_ERR_INVALID, "nb_world_read_behaviors: no behaviours set (nb_world_set_behaviors)");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  if (goals && w->O) NB_CUDA(cudaMemcpyAsync(goals, w->rvo.goal.get(), sizeof(double) * 2 * w->O, cudaMemcpyDeviceToDevice, st));
  if (draws && w->O) NB_CUDA(cudaMemcpyAsync(draws, w->rvo.draws.get(), sizeof(int32_t) * w->O, cudaMemcpyDeviceToDevice, st));
  return NB_OK;
}

int nb_world_scan(nb_world_t* w, int32_t B, float* ranges, float* velocity, int32_t* hit, void* stream) {
  if (int rc = world_ready(w, B, "nb_world_scan", true)) return rc;
  if (!ranges) return fail(NB_ERR_INVALID, "nb_world_scan: null ranges");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  // the dynamic shared-memory limit is an attribute of the kernel, shared by every handle of the process: set this handle's
  // size before each launch (another handle's nb_world_set_scenes may have set a smaller one)
  const bool map = w->maps.has_map;
  auto* kernel = w->range_std > 0.0
                     ? (w->ep.slots ? (map ? nb::world_scan_kernel<true, true, true> : nb::world_scan_kernel<false, true, true>)
                                    : (map ? nb::world_scan_kernel<true, false, true> : nb::world_scan_kernel<false, false, true>))
                     : (w->ep.slots ? (map ? nb::world_scan_kernel<true, true> : nb::world_scan_kernel<false, true>)
                                    : (map ? nb::world_scan_kernel<true, false> : nb::world_scan_kernel<false, false>));
  NB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(w->scan_smem, 1)));
  kernel<<<w->scan_grid, w->scan_threads, w->scan_smem, (cudaStream_t)stream>>>(world_params(w), world_map_params(w), w->max_circ, w->max_edges,
                                                                                w->max_redges, ranges, velocity, hit, world_noise_params(w, true));
  ++nb::launches;
  NB_CUDA(cudaGetLastError());
  return NB_OK;
}

int nb_world_step(nb_world_t* w, int32_t B, const float* action, int32_t* collided, int32_t* arrived, float* clearance, void* stream) {
  if (int rc = world_ready(w, B, "nb_world_step", true)) return rc;
  if (!action) return fail(NB_ERR_INVALID, "nb_world_step: null action");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  const nb::WorldParams prm = world_params(w);  // prm.B: the environments, or the slots in episode mode
  const bool ep = w->ep.slots > 0, map = w->maps.has_map, blocking = w->contact.has_block, contact = w->ocontact.has_contact;
  if (w->rvo.has_rvo) {  // reactive obstacles choose their velocities from the states at the start of the step
    const int grid = std::min(w->rvo.grid, prm.B);
    const size_t smem = w->rvo.smem;
    if (blocking) {
      auto* rvo = ep ? nb::world_rvo_block_kernel<true> : nb::world_rvo_block_kernel<false>;
      NB_CUDA(cudaFuncSetAttribute(rvo, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      rvo<<<grid, 32 * nb::kWorldRvoWarps, smem, (cudaStream_t)stream>>>(prm, world_rvo_params(w, action), world_map_params(w), world_block_params(w));
    } else {
      auto* rvo = ep ? nb::world_rvo_kernel<true> : nb::world_rvo_kernel<false>;
      NB_CUDA(cudaFuncSetAttribute(rvo, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      rvo<<<grid, 32 * nb::kWorldRvoWarps, smem, (cudaStream_t)stream>>>(prm, world_rvo_params(w, action));
    }
    ++nb::launches;
    NB_CUDA(cudaGetLastError());
  }
  // a CTA of up to 8 warps per E environments, a warp per robot
  const int E = nb::world_step_envs(w->K);
  const dim3 grid((prm.B + E - 1) / E), block(32 * std::min(E * w->K, nb::kWorldStepMaxWarps));
  const bool act = w->act.on;
  const nb::WorldNoiseParams nz = world_noise_params(w, false);
  if (contact) {  // the obstacles move one environment per warp, in row order; the step then leaves them where they are
    const int units = (prm.B + nb::kWorldContactWarps - 1) / nb::kWorldContactWarps;
    const size_t smem = sizeof(double) * nb::kWorldContactWarps * 6 * w->ocontact.max_n;
    auto* move = blocking ? (ep ? nb::world_contact_kernel<true, true> : nb::world_contact_kernel<true, false>)
                          : (ep ? nb::world_contact_kernel<false, true> : nb::world_contact_kernel<false, false>);
    move<<<units, 32 * nb::kWorldContactWarps, smem, (cudaStream_t)stream>>>(prm, world_map_params(w), world_block_params(w), world_contact_params(w));
    ++nb::launches;
    NB_CUDA(cudaGetLastError());
    if (act) {
      auto* kernel = ep ? (map ? nb::world_step_act_kernel<true, true, false, false> : nb::world_step_act_kernel<false, true, false, false>)
                        : (map ? nb::world_step_act_kernel<true, false, false, false> : nb::world_step_act_kernel<false, false, false, false>);
      kernel<<<grid, block, 0, (cudaStream_t)stream>>>(prm, world_map_params(w), nb::WorldBlockParams{}, nz, action, collided, arrived, clearance);
    } else {
      auto* kernel = ep ? (map ? nb::world_step_contact_kernel<true, true> : nb::world_step_contact_kernel<false, true>)
                        : (map ? nb::world_step_contact_kernel<true, false> : nb::world_step_contact_kernel<false, false>);
      kernel<<<grid, block, 0, (cudaStream_t)stream>>>(prm, world_map_params(w), action, collided, arrived, clearance);
    }
  } else if (act) {  // the step with the actuation stage: blocking maps, or the plain and episode kernels' variants
    auto* kernel = blocking ? (ep ? nb::world_step_act_kernel<true, true, true, true> : nb::world_step_act_kernel<true, false, true, true>)
                            : (ep ? (map ? nb::world_step_act_kernel<true, true, false, true> : nb::world_step_act_kernel<false, true, false, true>)
                                  : (map ? nb::world_step_act_kernel<true, false, false, true> : nb::world_step_act_kernel<false, false, false, true>));
    kernel<<<grid, block, 0, (cudaStream_t)stream>>>(prm, world_map_params(w), world_block_params(w), nz, action, collided, arrived, clearance);
  } else if (blocking) {
    auto* kernel = ep ? nb::world_step_block_kernel<true> : nb::world_step_block_kernel<false>;
    kernel<<<grid, block, 0, (cudaStream_t)stream>>>(prm, world_map_params(w), world_block_params(w), action, collided, arrived, clearance);
  } else {
    auto* kernel = ep ? (map ? nb::world_step_ep_kernel<true> : nb::world_step_ep_kernel<false>)
                      : (map ? nb::world_step_kernel<true> : nb::world_step_kernel<false>);
    kernel<<<grid, block, 0, (cudaStream_t)stream>>>(prm, world_map_params(w), action, collided, arrived, clearance);
  }
  ++nb::launches;
  NB_CUDA(cudaGetLastError());
  if (ep) {  // end the episodes of this step and hand out the next scenes
    const nb_world::Episodes& e = w->ep;
    nb::WorldEpisodeParams a;
    a.S = w->B; a.slots = e.slots; a.K = w->K; a.max_steps = e.max_steps;
    a.scene_of = e.scene_of.get(); a.live = e.live.get(); a.reset = e.reset.get(); a.t = e.t.get();
    a.next = e.count.get(); a.finished = e.count.get() + 1;
    a.collided = w->robots.collided.get(); a.arrived = w->robots.arrived.get(); a.clear = e.clear.get();
    a.r_col = e.r_col.get(); a.r_arr = e.r_arr.get(); a.r_astep = e.r_astep.get(); a.r_minclr = e.r_minclr.get();
    a.r_end = e.r_end.get(); a.r_reason = e.r_reason.get(); a.r_slot = e.r_slot.get();
    a.cmd = act ? w->robots.cmd.get() : nullptr;
    nb::world_advance_kernel<<<1, nb::kWorldAdvanceThreads, 0, (cudaStream_t)stream>>>(a);
    ++nb::launches;
    NB_CUDA(cudaGetLastError());
  }
  ++w->steps;
  return NB_OK;
}

int nb_world_read_state(nb_world_t* w, int32_t B, double* states, double* obstacles, int32_t* collided, int32_t* arrived, void* stream) {
  // episode mode: B = slots K reads the slot rows (a gather), B = S K the scenes' own rows (copies, like a plain world)
  const bool scenes = w && w->ep.slots && B == w->B * w->K;
  if (!scenes)
    if (int rc = world_ready(w, B, "nb_world_read_state", true)) return rc;
  NB_CUDA(cudaSetDevice(w->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const nb_world::Robots& r = w->robots;
  const double* obs = w->scenes.obs.get();
  if (w->ep.slots && !scenes) {
    if (obstacles && w->O) NB_CUDA(cudaMemcpyAsync(obstacles, obs, sizeof(double) * nb::kWorldObsCols * w->O, cudaMemcpyDeviceToDevice, st));
    if (!states && !collided && !arrived) return NB_OK;
    nb::world_gather_kernel<<<(B + 255) / 256, 256, 0, st>>>(w->ep.slots, w->K, w->ep.scene_of.get(), r.states.get(), r.collided.get(), r.arrived.get(),
                                                             states, collided, arrived);
    ++nb::launches;
    NB_CUDA(cudaGetLastError());
    return NB_OK;
  }
  if (states) NB_CUDA(cudaMemcpyAsync(states, r.states.get(), sizeof(double) * 3 * B, cudaMemcpyDeviceToDevice, st));
  if (obstacles && w->O) NB_CUDA(cudaMemcpyAsync(obstacles, obs, sizeof(double) * nb::kWorldObsCols * w->O, cudaMemcpyDeviceToDevice, st));
  if (collided) NB_CUDA(cudaMemcpyAsync(collided, r.collided.get(), sizeof(int32_t) * B, cudaMemcpyDeviceToDevice, st));
  if (arrived) NB_CUDA(cudaMemcpyAsync(arrived, r.arrived.get(), sizeof(int32_t) * B, cudaMemcpyDeviceToDevice, st));
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
  w->maps = {}; w->contact = {}; w->ocontact = {}; w->ep = {};  // the new starts need a new map check
  if (int rc = world_set_robots(w, B, K, robots, T, types, robot_type)) return rc;
  if (int rc = world_scan_shape(w, B)) return rc;
  if (w->rvo.beh)
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
  w->maps = {}; w->contact = {}; w->ocontact = {}; w->ep = {};
  const size_t words = (size_t)(table.back().off + (int64_t)table.back().H * table.back().words);
  nb_world::Maps m;
  auto upload = [&]() -> int {
    NB_CUDA(nb::alloc(m.table, table.size()));
    NB_CUDA(nb::alloc(m.bits, words));
    NB_CUDA(nb::alloc(m.env_map, (size_t)w->B));
    NB_CUDA(cudaMemcpy(m.table.get(), table.data(), sizeof(nb::WorldMap) * table.size(), cudaMemcpyHostToDevice));
    NB_CUDA(cudaMemcpy(m.bits.get(), bits, sizeof(uint32_t) * words, cudaMemcpyHostToDevice));
    NB_CUDA(cudaMemcpy(m.env_map.get(), env_map, sizeof(int32_t) * w->B, cudaMemcpyHostToDevice));
    return NB_OK;
  };
  if (int rc = upload()) {  // the handle stays usable, without maps
    cudaGetLastError();
    if (int rc2 = world_scan_shape(w, w->B)) return rc2;
    return rc;
  }
  m.has_map = std::any_of(env_map, env_map + w->B, [](int32_t e) { return e >= 0; });
  m.window = window;
  m.h_table = std::move(table);
  m.h_bits.assign(bits, bits + words);
  m.h_env_map.assign(env_map, env_map + w->B);
  w->maps = std::move(m);
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
  w->ep = {};
  const size_t SK = (size_t)S * K, BK = (size_t)slots * K;
  std::vector<int32_t> scene_of(slots), slot(S, -1), minus(SK, -1), ones(slots, 1);
  for (int b = 0; b < slots; ++b) scene_of[b] = slot[b] = b;
  const int32_t count[2] = {slots, 0};  // the next scene, episodes finished
  std::vector<float> inf(SK, INFINITY);
  nb_world::Episodes ep;
  auto upload = [&]() -> int {
    NB_CUDA(nb::alloc(ep.scene_of, slots)); NB_CUDA(nb::alloc(ep.live, slots)); NB_CUDA(nb::alloc(ep.reset, slots));
    NB_CUDA(nb::alloc(ep.t, slots)); NB_CUDA(nb::alloc(ep.count, 2));
    NB_CUDA(nb::alloc(ep.clear, BK));
    NB_CUDA(nb::alloc(ep.r_col, SK)); NB_CUDA(nb::alloc(ep.r_arr, SK)); NB_CUDA(nb::alloc(ep.r_astep, SK)); NB_CUDA(nb::alloc(ep.r_minclr, SK));
    NB_CUDA(nb::alloc(ep.r_end, S)); NB_CUDA(nb::alloc(ep.r_reason, S)); NB_CUDA(nb::alloc(ep.r_slot, S));
    auto up = [](auto& d, const auto* h, size_t n) { return cudaMemcpy(d.get(), h, n * sizeof(*h), cudaMemcpyHostToDevice); };
    NB_CUDA(up(ep.scene_of, scene_of.data(), slots));
    NB_CUDA(up(ep.live, ones.data(), slots));
    NB_CUDA(up(ep.reset, ones.data(), slots));  // every slot has just taken its first scene
    NB_CUDA(cudaMemset(ep.t.get(), 0, slots * sizeof(int32_t)));
    NB_CUDA(up(ep.count, count, 2));
    NB_CUDA(cudaMemset(ep.r_col.get(), 0, SK * sizeof(int32_t)));
    NB_CUDA(cudaMemset(ep.r_arr.get(), 0, SK * sizeof(int32_t)));
    NB_CUDA(up(ep.r_astep, minus.data(), SK));
    NB_CUDA(up(ep.r_minclr, inf.data(), SK));
    NB_CUDA(cudaMemset(ep.r_end.get(), 0, S * sizeof(int32_t)));
    NB_CUDA(cudaMemset(ep.r_reason.get(), 0, S * sizeof(int32_t)));
    NB_CUDA(up(ep.r_slot, slot.data(), S));
    NB_CUDA(cudaMemset(w->robots.cmd.get(), 0, SK * 2 * sizeof(double)));  // every scene starts from a zero command
    NB_CUDA(cudaDeviceSynchronize());
    return NB_OK;
  };
  if (int rc = upload()) {  // the handle stays usable as a plain world
    cudaGetLastError();
    return rc;
  }
  ep.slots = slots; ep.max_steps = max_steps;
  w->ep = std::move(ep);
  w->steps = 0;
  return NB_OK;
}

int nb_world_read_episodes(nb_world_t* w, int32_t S, int32_t* collided, int32_t* arrived, int32_t* arrive_step, float* min_clearance, int32_t* end_step,
                           int32_t* reason, int32_t* slot, int32_t* scene_of, int32_t* reset, int32_t* finished, void* stream) {
  if (int rc = world_ready(w, S, "nb_world_read_episodes")) return rc;
  const nb_world::Episodes& ep = w->ep;
  if (!ep.slots) return fail(NB_ERR_INVALID, "nb_world_read_episodes: not in episode mode (nb_world_set_episodes)");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t SK = (size_t)S * w->K;
  auto cp = [&](void* dst, const void* src, size_t bytes) { return dst ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st) : cudaSuccess; };
  NB_CUDA(cp(collided, ep.r_col.get(), SK * sizeof(int32_t)));
  NB_CUDA(cp(arrived, ep.r_arr.get(), SK * sizeof(int32_t)));
  NB_CUDA(cp(arrive_step, ep.r_astep.get(), SK * sizeof(int32_t)));
  NB_CUDA(cp(min_clearance, ep.r_minclr.get(), SK * sizeof(float)));
  NB_CUDA(cp(end_step, ep.r_end.get(), S * sizeof(int32_t)));
  NB_CUDA(cp(reason, ep.r_reason.get(), S * sizeof(int32_t)));
  NB_CUDA(cp(slot, ep.r_slot.get(), S * sizeof(int32_t)));
  NB_CUDA(cp(scene_of, ep.scene_of.get(), ep.slots * sizeof(int32_t)));
  NB_CUDA(cp(reset, ep.reset.get(), ep.slots * sizeof(int32_t)));
  NB_CUDA(cp(finished, ep.count.get() + 1, sizeof(int32_t)));
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
  if (!w->maps.table) return fail(NB_ERR_INVALID, "nb_world_set_map_contact: no maps set (nb_world_set_maps)");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  const int O = w->O;
  nb_world::Behaviors& rvo = w->rvo;
  std::vector<double> obs((size_t)nb::kWorldObsCols * O), beh;
  if (O) NB_CUDA(cudaMemcpy(obs.data(), w->scenes.obs.get(), sizeof(double) * obs.size(), cudaMemcpyDeviceToHost));  // the current centres
  if (rvo.beh && O) {
    beh.resize((size_t)nb::kWorldBehCols * O);
    NB_CUDA(cudaMemcpy(beh.data(), rvo.beh.get(), sizeof(double) * beh.size(), cudaMemcpyDeviceToHost));
  }
  if (int rc = world_check_contact(&w->cfg, B, w->h_obs_begin.data(), obs.data(), w->h_vert_begin.data(), w->h_vertices.data(), w->h_kind.data(),
                                   beh.empty() ? nullptr : beh.data(), w->maps.h_table, w->maps.h_bits.data(), w->maps.h_env_map.data(), flags))
    return rc;
  w->contact = {}; w->ocontact = {}; w->ep = {};
  // a wandering obstacle without an explicit goal in a blocking environment starts from goal = its centre and draw 0, so that its
  // first goal is drawn on the device through the map test
  std::vector<double> goal;
  std::vector<int32_t> draws;
  bool reset = false;
  if (!beh.empty()) {
    goal.resize(2 * (size_t)O); draws.resize(O);
    NB_CUDA(cudaMemcpy(goal.data(), rvo.goal.get(), sizeof(double) * goal.size(), cudaMemcpyDeviceToHost));
    NB_CUDA(cudaMemcpy(draws.data(), rvo.draws.get(), sizeof(int32_t) * O, cudaMemcpyDeviceToHost));
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
  nb_world::Contact c;
  auto upload = [&]() -> int {
    NB_CUDA(nb::alloc(c.block, (size_t)B));
    NB_CUDA(nb::alloc(c.bounces, (size_t)O));
    NB_CUDA(nb::alloc(c.bounced, (size_t)O));
    NB_CUDA(cudaMemcpy(c.block.get(), flags, sizeof(int32_t) * B, cudaMemcpyHostToDevice));
    NB_CUDA(cudaMemset(c.bounces.get(), 0, sizeof(int32_t) * std::max(O, 1)));
    NB_CUDA(cudaMemset(c.bounced.get(), 0, sizeof(int32_t) * std::max(O, 1)));
    if (reset) NB_CUDA(cudaMemcpy(rvo.goal.get(), goal.data(), sizeof(double) * goal.size(), cudaMemcpyHostToDevice));
    if (reset) NB_CUDA(cudaMemcpy(rvo.draws.get(), draws.data(), sizeof(int32_t) * O, cudaMemcpyHostToDevice));
    NB_CUDA(cudaDeviceSynchronize());
    return NB_OK;
  };
  if (int rc = upload()) {  // no contact flags
    cudaGetLastError();
    return rc;
  }
  c.has_block = std::any_of(flags, flags + B, [](int32_t f) { return f != 0; });
  w->contact = std::move(c);
  return NB_OK;
}

int nb_world_read_map_contact(nb_world_t* w, int32_t O, int32_t* bounces, void* stream) {
  if (!w) return fail(NB_ERR_INVALID, "nb_world_read_map_contact: null handle");
  if (!w->contact.bounces) return fail(NB_ERR_INVALID, "nb_world_read_map_contact: no map contact set (nb_world_set_map_contact)");
  if (O != w->O) return fail(NB_ERR_INVALID, "nb_world_read_map_contact: O = %d but the scenes have %d obstacles", O, w->O);
  if (!bounces) return fail(NB_ERR_INVALID, "nb_world_read_map_contact: null bounces");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  if (O) NB_CUDA(cudaMemcpyAsync(bounces, w->contact.bounces.get(), sizeof(int32_t) * O, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return NB_OK;
}


int nb_world_check_obstacle_contact(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obstacles, const int32_t* vert_begin,
                                    const double* vertices, const double* envs, const int32_t* obs_kind, const double* behaviors, const int32_t* flags) {
  if (int rc = world_check_scenes(cfg, B, obs_begin, obstacles, vert_begin, vertices, envs, obs_kind, nullptr, nullptr, nullptr, nullptr)) return rc;
  if (behaviors)
    if (int rc = world_check_behaviors(cfg, B, obs_begin, obstacles, envs, behaviors)) return rc;
  return world_check_obstacle_contact(B, obs_begin, obstacles, vert_begin, vertices, obs_kind, behaviors, flags);
}

int nb_world_set_obstacle_contact(nb_world_t* w, int32_t B, const int32_t* flags) {
  if (int rc = world_ready(w, B, "nb_world_set_obstacle_contact")) return rc;
  NB_CUDA(cudaSetDevice(w->cfg.device));
  const int O = w->O;
  std::vector<double> obs((size_t)nb::kWorldObsCols * O), beh;
  if (O) NB_CUDA(cudaMemcpy(obs.data(), w->scenes.obs.get(), sizeof(double) * obs.size(), cudaMemcpyDeviceToHost));  // the current centres
  if (w->rvo.beh && O) {
    beh.resize((size_t)nb::kWorldBehCols * O);
    NB_CUDA(cudaMemcpy(beh.data(), w->rvo.beh.get(), sizeof(double) * beh.size(), cudaMemcpyDeviceToHost));
  }
  if (int rc = world_check_obstacle_contact(B, w->h_obs_begin.data(), obs.data(), w->h_vert_begin.data(), w->h_vertices.data(), w->h_kind.data(),
                                            beh.empty() ? nullptr : beh.data(), flags))
    return rc;
  w->ocontact = {}; w->ep = {};
  nb_world::ObstacleContact c;
  auto upload = [&]() -> int {
    NB_CUDA(nb::alloc(c.flag, (size_t)B));
    NB_CUDA(nb::alloc(c.bounces, (size_t)O));
    NB_CUDA(cudaMemcpy(c.flag.get(), flags, sizeof(int32_t) * B, cudaMemcpyHostToDevice));
    NB_CUDA(cudaMemset(c.bounces.get(), 0, sizeof(int32_t) * std::max(O, 1)));
    NB_CUDA(cudaDeviceSynchronize());
    return NB_OK;
  };
  if (int rc = upload()) {  // no contact flags
    cudaGetLastError();
    return rc;
  }
  for (int b = 0; b < B; ++b) c.max_n = std::max(c.max_n, w->h_obs_begin[b + 1] - w->h_obs_begin[b]);
  c.has_contact = std::any_of(flags, flags + B, [](int32_t f) { return f != 0; });
  w->ocontact = std::move(c);
  return NB_OK;
}

int nb_world_read_obstacle_contact(nb_world_t* w, int32_t O, int32_t* bounces, void* stream) {
  if (!w) return fail(NB_ERR_INVALID, "nb_world_read_obstacle_contact: null handle");
  if (!w->ocontact.bounces) return fail(NB_ERR_INVALID, "nb_world_read_obstacle_contact: no obstacle contact set (nb_world_set_obstacle_contact)");
  if (O != w->O) return fail(NB_ERR_INVALID, "nb_world_read_obstacle_contact: O = %d but the scenes have %d obstacles", O, w->O);
  if (!bounces) return fail(NB_ERR_INVALID, "nb_world_read_obstacle_contact: null bounces");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  if (O) NB_CUDA(cudaMemcpyAsync(bounces, w->ocontact.bounces.get(), sizeof(int32_t) * O, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return NB_OK;
}

int nb_world_set_actuation(nb_world_t* w, int32_t num_types, const nb_world_actuation* per_type, uint64_t seed) {
  if (!w) return fail(NB_ERR_INVALID, "nb_world_set_actuation: null handle");
  if (int rc = world_check_actuation(w, num_types, per_type)) return rc;
  NB_CUDA(cudaSetDevice(w->cfg.device));
  const double inf = INFINITY;
  const double def[nb::kWorldActCols] = {-inf, -inf, inf, inf, inf, inf, 0.0, 0.0, 0.0, 0.0};
  std::vector<double> table((size_t)nb::kWorldMaxRobotTypes * nb::kWorldActCols);
  for (int t = 0; t < nb::kWorldMaxRobotTypes; ++t) {
    double* row = table.data() + (size_t)t * nb::kWorldActCols;
    if (t < num_types) {
      const nb_world_actuation& a = per_type[t];
      const double r[nb::kWorldActCols] = {a.vel_min[0], a.vel_min[1], a.vel_max[0], a.vel_max[1], a.acce[0], a.acce[1],
                                           a.alpha[0], a.alpha[1], a.alpha[2], a.alpha[3]};
      std::copy(r, r + nb::kWorldActCols, row);
    } else {
      std::copy(def, def + nb::kWorldActCols, row);
    }
  }
  if (!w->act.act) NB_CUDA(nb::alloc(w->act.act, table.size()));
  NB_CUDA(cudaMemcpy(w->act.act.get(), table.data(), sizeof(double) * table.size(), cudaMemcpyHostToDevice));
  w->act.seed = seed;
  w->act.on = true;
  return NB_OK;
}

int nb_world_set_lidar_noise(nb_world_t* w, double range_min, double range_std, uint64_t seed) {
  if (!w) return fail(NB_ERR_INVALID, "nb_world_set_lidar_noise: null handle");
  if (!(std::isfinite(range_std) && range_std >= 0.0))
    return fail(NB_ERR_INVALID, "nb_world_set_lidar_noise: range_std = %g must be finite and >= 0", range_std);
  if (!(range_min >= 0.0 && range_min < w->cfg.range_max))
    return fail(NB_ERR_INVALID, "nb_world_set_lidar_noise: range_min = %g outside [0, range_max = %g)", range_min, w->cfg.range_max);
  w->range_min = range_min; w->range_std = range_std; w->lidar_seed = seed;
  return NB_OK;
}

int nb_world_read_commands(nb_world_t* w, int32_t N, double* cmd_prev, void* stream) {
  if (!w) return fail(NB_ERR_INVALID, "nb_world_read_commands: null handle");
  if (!w->B) return fail(NB_ERR_INVALID, "nb_world_read_commands: no scenes set (nb_world_set_scenes)");
  if (N != w->B * w->K)
    return fail(NB_ERR_INVALID, "nb_world_read_commands: N = %d but the world has %d %s x %d robots (N = %d)", N, w->B, w->ep.slots ? "scenes" : "environments",
                w->K, w->B * w->K);
  if (!cmd_prev) return fail(NB_ERR_INVALID, "nb_world_read_commands: null cmd_prev");
  NB_CUDA(cudaSetDevice(w->cfg.device));
  NB_CUDA(cudaMemcpyAsync(cmd_prev, w->robots.cmd.get(), sizeof(double) * 2 * (size_t)N, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return NB_OK;
}

}  // extern "C"
