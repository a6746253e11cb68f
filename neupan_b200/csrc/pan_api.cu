// C-ABI of the PAN hot path (include/neupan_b200.h): handle, workspaces, launch logic.  The DUNE kernels are launched by dune_tc.cu,
// the NRMP kernels by nrmp.cu.  Also the library-wide error text and launch counter.
// No torch, no C++ types across the boundary.  One handle = one (process, GPU); not thread-safe.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <chrono>
#include <cstring>
#include <memory>
#include <new>
#include <vector>

#include "host_common.h"
#include "dune_common.cuh"
#include "dune_table_kernel.cuh"
#include "nrmp_common.cuh"

using nb::fail;

struct nb_pan {
  nb_pan_config cfg;
  nb::Geometry geo;
  int sm_count = 0;
  int max_smem_optin = 0;
  // device buffers
  nb::DeviceArray<float> d_weights;
  nb::DeviceArray<unsigned char> d_tc_image;  // wgmma operand image of the warpgroup DUNE kernels
  int tc_flags = 0;                           // build_tc_image(): bit 0 = bounded tanh arguments
  nb::DeviceArray<unsigned char> d_tc_screen; // operand image of the screening network (NB_OPT_DUNE_KERNEL = 4)
  nb::DeviceArray<int32_t> cand_idx, cand_cnt, flag_list, flag_count, refine_list;
  nb::DeviceArray<float> cand_dt, cand_rad;
  nb::DeviceArray<unsigned> screen_stats;
  float c_mu = 0.012f;                  // bound on the screening network's |mu~ - mu|: set by calibrate_screen() to 4 x the largest error
                                        // measured for THIS checkpoint and polygon (NB_SCREEN_CMU overrides; DESIGN.md 3.1)
  bool screen_calibrated = false;
  float screen_cal_ratio = 0.f;
  bool cmu_override = false;            // NB_SCREEN_CMU is set: every point gets the radius c_mu sum_e |G_e p0 - h_e| + 1e-4 (network screen)
  int screen_table = 1;                 // NB_OPT_DUNE_SCREEN_TABLE: the mma.sync screen looks distances up in the table below
  nb::DeviceArray<float4> tab_cell;     // distance table (dune_table_kernel.cuh), built once per handle by build_screen_table()
  nb::DeviceArray<float> tab_rad;
  nb::DeviceArray<uint32_t> tab_coarse; // its coarse bound table (dune_table_coarse_kernel), tab_cn x tab_cn
  int tab_n = 0, tab_cn = 0;
  int screen_coarse = 1;                // NB_SCREEN_COARSE=0 (developer switch, read at create): every item takes the one-level table path
  nb::DeviceArray<unsigned> coarse_stats;  // survivors of the coarse pass and items that took the one-level path (nb_pan_read_screen_coarse)
  float tab_h = 0.f, tab_half = 0.f, tab_ratio = 0.f, tab_ms = 0.f;
  bool tab_built = false;               // built (and kept, or freed as not accurate enough: tab_cell empty)
  int dune_variant = 2;              // NB_OPT_DUNE_KERNEL: 2 = the exact wgmma kernel on every point, 4 = screening pipeline
  int overlap = 1;                   // NB_OPT_OVERLAP: number of env sub-batches pipelined on internal streams
  nb::Stream streams[4];
  nb::Event ev_fork, ev_join[4];
  // host-input entry points: uploads run on copy_stream in env chunks; ev_chunk[c] = chunk c (and everything before it) has landed
  static constexpr int kMaxChunks = 8;
  nb::Stream copy_stream;
  nb::Event ev_chunk[kMaxChunks], ev_inputs_free;
  int h2d_chunks = 4;               // NB_H2D_CHUNKS (developer switch, read at create); 1 = no overlap
  nb::DeviceArray<float> sel_mu, sel_lam, sel_pts, sel_dist;
  nb::DeviceArray<int32_t> sel_count;
  nb::DeviceArray<float> prev_s, prev_u, prev_mu, prev_lam;
  nb::DeviceArray<int32_t> prev_count, prev_valid, active, iters, status, ipm_it;
  nb::DeviceArray<float> min_dist;
  // differentiable mode (NB_OPT_DIFFERENTIABLE): adjoint records of every (iteration, env) solve for `iters` iterations + gradient
  // workspaces; allocated as a whole or not at all
  struct Adjoint {
    int iters = 0;
    nb::DeviceArray<double> rec, gs, gu, gd, gtheta;
    nb::DeviceArray<int32_t> valid;
  };
  int differentiable = 0;
  Adjoint adj;
  nb::DeviceArray<int> work_counters;  // dynamic env -> warp assignment of the NRMP kernel, one counter per internal stream
  int dune_skip_t0 = 1;             // NB_OPT_DUNE_SKIP_T0: PAN iterations k > 0 keep the step-0 items of iteration 0 (screening variant)
  int screen_mma = 1;               // NB_OPT_DUNE_SCREEN_MMA: screening pass on mma.sync (N <= 1024) instead of wgmma
  int nrmp_defer_stop_min = 256;    // NB_NRMP_DEFER_STOP_MIN (developer switch, read at create): smallest batch whose stop criterion runs as its own kernel
  int nrmp_dynamic = 1;             // NB_NRMP_STATIC=1 (developer switch, read at create) turns the persistent-warp schedule off
  nb::DeviceArray<float> warm;      // NRMP warm-start records, nrmp_warm_floats(T, M) per environment
  nb::DeviceArray<int32_t> warm_valid;
  int nrmp_warm = 0;                // NB_OPT_NRMP_WARM (off by default: see DESIGN.md 3.2)
  double nrmp_gap_tol = 1e-12;      // NB_NRMP_GAP_TOL (developer switch, read once at create)
  int warm_check_it = 12;           // NB_NRMP_RESTART_IT / NB_NRMP_RESTART_GAP (developer switches): early cold restart of a warm start
  double warm_check_gap = 1e-5;
  // staging for the host-pointer entry point
  nb::DeviceArray<float> h_in, h_out;  // device staging
  size_t h_in_floats = 0, h_out_floats = 0;
  nb::DeviceArray<int32_t> h_np;
  nb::DeviceArray<int32_t> h_io;
};

namespace {

int check_forward_args(const nb_pan* p, int B, int N) {
  if (!p) return fail(NB_ERR_INVALID, "null handle");
  if (B <= 0) return fail(NB_ERR_INVALID, "B must be positive (got %d)", B);
  if (B > p->cfg.max_envs) return fail(NB_ERR_CAPACITY, "B=%d exceeds max_envs=%d", B, p->cfg.max_envs);
  if (N < 0) return fail(NB_ERR_INVALID, "N must be >= 0");
  if (N > p->cfg.max_points) return fail(NB_ERR_CAPACITY, "N=%d exceeds max_points=%d", N, p->cfg.max_points);
  return NB_OK;
}

// The DUNE parameters of what the handle owns: weights, geometry, shapes, the screening state and the bases of its per-environment
// buffers.  Callers add the inputs, B, N, active / min_dist and the distance table, and move the per-environment pointers with dune_offset.
nb::DuneParams dune_params(const nb_pan* p) {
  const nb_pan_config& c = p->cfg;
  nb::DuneParams d{};
  d.weights = p->d_weights.get(); d.geo = p->geo;
  d.T = c.receding; d.M = c.nrmp_max_num; d.dt = (float)c.step_time;
  d.c_mu = p->c_mu; d.screen_stats = p->screen_stats.get(); d.screen_mma = p->screen_mma; d.coarse_stats = p->coarse_stats.get();
  d.sel_mu = p->sel_mu.get(); d.sel_lam = p->sel_lam.get(); d.sel_pts = p->sel_pts.get(); d.sel_dist = p->sel_dist.get(); d.sel_count = p->sel_count.get();
  d.cand_idx = p->cand_idx.get(); d.cand_dt = p->cand_dt.get(); d.cand_cnt = p->cand_cnt.get(); d.cand_rad = p->cand_rad.get();
  d.flag_list = p->flag_list.get(); d.flag_count = p->flag_count.get(); d.refine_list = p->refine_list.get();
  return d;
}

// Moves every per-environment pointer of d (the null ones stay null) on by `off` environments.  flag_count (a slot per stream),
// screen_stats, the weights and the distance table are shared by the whole batch and stay where they are.
void dune_offset(nb::DuneParams& d, size_t off) {
  const size_t T1 = (size_t)d.T + 1, M = (size_t)d.M, E = (size_t)d.geo.E, N = (size_t)d.N, C = nb::kCandMax;
  auto adv = [off](auto*& q, size_t per_env) { if (q) q += off * per_env; };
  adv(d.nom_s, 3 * T1); adv(d.points, 2 * N); adv(d.velocities, 2 * N); adv(d.num_points, 1); adv(d.active, 1);
  adv(d.sel_mu, T1 * M * E); adv(d.sel_lam, T1 * M * 2); adv(d.sel_pts, T1 * M * 2); adv(d.sel_dist, T1 * M); adv(d.sel_count, 1);
  adv(d.min_dist, 1);
  adv(d.cand_idx, T1 * C); adv(d.cand_dt, T1 * C); adv(d.cand_cnt, T1); adv(d.cand_rad, T1 * C);
  adv(d.flag_list, T1); adv(d.refine_list, 2 * T1);
}

// The NRMP parameters of the handle's configuration (nb_pan_config, and the developer switches read at create); callers add the
// tensors and B
nb::NrmpParams nrmp_params(const nb_pan* p) {
  const nb_pan_config& c = p->cfg;
  nb::NrmpParams prm{};
  prm.T = c.receding; prm.M = c.nrmp_max_num; prm.E = c.edge_dim; prm.kin = c.kinematics;
  prm.max_ipm_iter = 60;
  prm.gap_tol = p->nrmp_gap_tol;
  prm.warm_check_it = p->warm_check_it; prm.warm_check_gap = p->warm_check_gap;
  prm.iter_threshold = c.iter_threshold;
  prm.dt = c.step_time; prm.L = c.wheelbase;
  for (int i = 0; i < 3; ++i) prm.q[i] = c.q_s[i];
  prm.p_u = c.p_u; prm.eta = c.eta; prm.d_max = c.d_max; prm.d_min = c.d_min;
  prm.ro = c.ro_obs; prm.bk = c.bk;
  for (int i = 0; i < 2; ++i) {
    prm.speed[i] = c.max_speed[i];
    prm.acce[i] = c.max_acce[i] * c.step_time;
  }
  for (int e = 0; e < nb::kMaxEdges; ++e) prm.h[e] = p->geo.h[e];
  return prm;
}

// what an NRMP launch on the internal stream `counter_slot` (0: the caller's stream) borrows from the handle
nb::NrmpLaunch nrmp_launch(const nb_pan* p, int counter_slot) {
  return {p->sm_count, p->max_smem_optin, p->nrmp_defer_stop_min, p->nrmp_dynamic, p->work_counters.get() + counter_slot};
}

// Screening bound of this handle: the screen and the exact network evaluate the same 32-point items (points uniform in the square the
// reference trains DUNE on, [-25, 25]^2, and in [-6, 6]^2 around the robot, identity frame) and the refine kernel's statistics give
// max |d~ - d| / sum_e |G_e p - h_e| over every point; c_mu = 4 x that, clamped to [0.004, 0.05].
int calibrate_screen(nb_pan* p, cudaStream_t st) {
  const nb_pan_config& c = p->cfg;
  const int T1 = c.receding + 1, N = 32;
  int Bc = c.max_envs < 512 ? c.max_envs : 512;
  const int rounds = (4096 + Bc * T1 - 1) / (Bc * T1) < 1 ? 1 : (4096 + Bc * T1 - 1) / (Bc * T1);
  std::vector<float> pts((size_t)Bc * 2 * N), ns((size_t)Bc * 3 * T1, 0.f);
  nb::DeviceArray<float> d_pts, d_ns, d_md;
  NB_CUDA(nb::alloc(d_pts, pts.size()));
  NB_CUDA(nb::alloc(d_ns, ns.size()));
  NB_CUDA(nb::alloc(d_md, (size_t)Bc));
  NB_CUDA(cudaMemcpyAsync(d_ns.get(), ns.data(), ns.size() * sizeof(float), cudaMemcpyHostToDevice, st));
  unsigned saved[4];
  NB_CUDA(cudaStreamSynchronize(st));
  NB_CUDA(cudaMemcpy(saved, p->screen_stats.get(), sizeof(saved), cudaMemcpyDeviceToHost));
  NB_CUDA(cudaMemset(p->screen_stats.get(), 0, sizeof(saved)));
  unsigned long long rng = 0x9E3779B97F4A7C15ull;
  auto uni = [&]() { rng = rng * 6364136223846793005ull + 1442695040888963407ull; return (float)((rng >> 40) * (1.0 / 16777216.0)); };
  int rc = NB_OK;
  for (int r = 0; r < (rounds > 16 ? 16 : rounds) && rc == NB_OK; ++r) {
    for (int b = 0; b < Bc; ++b) {
      const float R = ((b + r) & 1) ? 25.f : 6.f;
      for (int i = 0; i < N; ++i) { pts[((size_t)b * 2) * N + i] = R * (2.f * uni() - 1.f); pts[((size_t)b * 2 + 1) * N + i] = R * (2.f * uni() - 1.f); }
    }
    cudaError_t e = cudaMemcpyAsync(d_pts.get(), pts.data(), pts.size() * sizeof(float), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) { rc = fail(NB_ERR_CUDA, "calibrate_screen: %s", cudaGetErrorString(e)); break; }
    nb::DuneParams prm = dune_params(p);  // no distance table: this measures the screening network
    prm.nom_s = d_ns.get(); prm.points = d_pts.get(); prm.min_dist = d_md.get();
    prm.B = Bc; prm.N = N; prm.calibrate = 1;
    for (int shape = 0; shape < 2 && rc == NB_OK; ++shape) {  // both screening kernels (wgmma / mma.sync): the bound holds whichever option is set later
      prm.screen_mma = shape;
      rc = nb::launch_dune_tc(prm, p->d_tc_image.get(), p->d_tc_screen.get(), p->tc_flags, true, p->sm_count, p->max_smem_optin, st);
      if (rc == NB_OK && cudaStreamSynchronize(st) != cudaSuccess) rc = fail(NB_ERR_CUDA, "calibrate_screen: kernel failed");
    }
  }
  if (rc == NB_OK) {
    unsigned h[4];
    NB_CUDA(cudaMemcpy(h, p->screen_stats.get(), sizeof(h), cudaMemcpyDeviceToHost));
    float ratio;
    memcpy(&ratio, &h[0], 4);
    p->screen_cal_ratio = ratio;
    float cm = 4.f * ratio;
    p->c_mu = cm < 0.008f ? 0.008f : (cm > 0.05f ? 0.05f : cm);
    if (const char* e = getenv("NB_SCREEN_CMU")) p->c_mu = (float)atof(e);
    p->screen_calibrated = true;
  }
  cudaMemcpy(p->screen_stats.get(), saved, sizeof(saved), cudaMemcpyHostToDevice);
  return rc;
}

// The distance table of the mma.sync screen (dune_table_kernel.cuh): cells of h metres over [-half, half]^2 of the robot frame,
// rounded up to whole cells.  The defaults h = 0.04, half = 16.384 cover clouds of up to 10 m around the start, a robot displacement of
// up to ~4 m and a point flow of up to 1.5 m over the horizon in 13.4 MB; points outside take the screening network.
// NB_SCREEN_TABLE_GRID="h,half" (metres) overrides both.  The table is kept only where it is at least twice as accurate as the
// handle's screening bound: largest |table - network| / sum_e |G_e p - h_e| on the fine samples <= c_mu / 2, so that the statistic
// nb_pan_read_screen_stats compares with c_mu keeps its margin.  Otherwise (at 4 cm: the acker and polygon checkpoints, whose ReLU
// kinks near the polygon give 7e-3 and 1e-2) it is freed and the handle keeps the network screen.
int build_screen_table(nb_pan* p) {
  float h = 0.04f, half = 16.384f;
  if (const char* e = getenv("NB_SCREEN_TABLE_GRID"))
    if (sscanf(e, "%f,%f", &h, &half) != 2 || !(h >= 1e-3f) || !(half > 0.f) || !(half < 1e3f))
      return fail(NB_ERR_INVALID, "NB_SCREEN_TABLE_GRID takes \"h,half\" in metres, h >= 0.001 (got \"%s\")", e);
  const long long n = (long long)ceilf(2.f * half / h);
  if (n > 4096) return fail(NB_ERR_INVALID, "NB_SCREEN_TABLE_GRID: %lld cells per side (at most 4096)", n);
  half = 0.5f * (float)n * h;
  const long long m = nb::kTableSub * n + 1;
  const auto t0 = std::chrono::steady_clock::now();
  NB_CUDA(cudaDeviceSynchronize());
  nb::DeviceArray<float> fine;
  nb::DeviceArray<unsigned> d_ratio;
  NB_CUDA(nb::alloc(fine, (size_t)(m * m)));
  NB_CUDA(nb::alloc(d_ratio, (size_t)1));
  if (!p->tab_cell) NB_CUDA(nb::alloc(p->tab_cell, (size_t)(n * n)));
  if (!p->tab_rad) NB_CUDA(nb::alloc(p->tab_rad, (size_t)(n * n)));
  const long long cn = (n + (1 << nb::kCoarseLog) - 1) >> nb::kCoarseLog;
  if (!p->tab_coarse) NB_CUDA(nb::alloc(p->tab_coarse, (size_t)(cn * cn)));
  NB_CUDA(cudaMemset(d_ratio.get(), 0, sizeof(unsigned)));
  const float hs = h / nb::kTableSub;
  nb::dune_table_sample_kernel<<<p->sm_count * 16, 128>>>(p->d_weights.get(), p->geo, (int)m, half, hs, fine.get());
  nb::dune_table_cell_kernel<<<p->sm_count * 8, 128>>>(fine.get(), (int)n, half, hs, p->geo, p->tab_cell.get(), p->tab_rad.get(), d_ratio.get());
  nb::dune_table_coarse_kernel<<<p->sm_count, 128>>>(p->tab_cell.get(), p->tab_rad.get(), (int)n, (int)cn, p->tab_coarse.get());
  NB_CUDA(cudaGetLastError());
  NB_CUDA(cudaDeviceSynchronize());
  unsigned r = 0;
  NB_CUDA(cudaMemcpy(&r, d_ratio.get(), sizeof(r), cudaMemcpyDeviceToHost));
  fine.reset();
  d_ratio.reset();
  memcpy(&p->tab_ratio, &r, 4);
  p->tab_n = (int)n; p->tab_cn = (int)cn; p->tab_h = h; p->tab_half = half; p->tab_built = true;
  if (!(2.f * p->tab_ratio <= p->c_mu)) {
    p->tab_cell.reset();
    p->tab_rad.reset();
    p->tab_coarse.reset();
  }
  p->tab_ms = (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return NB_OK;
}

// the table goes to the screen only where it is meant to be used; without it every point runs the screening network
void set_screen_table(const nb_pan* p, nb::DuneParams& prm) {
  const bool on = p->screen_table && !p->cmu_override && p->tab_cell;
  prm.tab_cell = on ? p->tab_cell.get() : nullptr;
  prm.tab_rad = p->tab_rad.get();
  prm.tab_n = p->tab_n;
  prm.tab_half = p->tab_half;
  prm.tab_inv_h = on ? 1.f / p->tab_h : 0.f;
  prm.tab_coarse = on && p->screen_coarse ? p->tab_coarse.get() : nullptr;
  prm.tab_cn = p->tab_cn;
}

__global__ void init_run_kernel(int B, int32_t* active, int32_t* iters, int32_t* status, float* min_dist, int32_t* sel_count, int32_t* warm_valid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) {
    active[i] = 1; iters[i] = 0; status[i] = 0;
    warm_valid[i] = 0;  // the first NRMP solve of a forward() is cold: results do not depend on earlier calls
    min_dist[i] = __int_as_float(0x7f800000);
    sel_count[i] = 0;
  }
}

// nb_pan_reset_envs_async: the state nb_pan_reset_state_async clears, for the environments whose mask is non-zero
__global__ void reset_envs_kernel(int B, const int32_t* mask, int32_t* prev_valid, int32_t* prev_count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B && mask[i] != 0) { prev_valid[i] = 0; prev_count[i] = 0; }
}

__global__ void finish_run_kernel(int B, const int32_t* iters, const int32_t* status, const float* min_dist,
                                  int32_t* out_iters, int32_t* out_status, float* out_min_dist) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) {
    if (out_iters) out_iters[i] = iters[i];
    if (out_status) out_status[i] = status[i];
    if (out_min_dist) out_min_dist[i] = min_dist[i];
  }
}

thread_local char g_err[512] = "";

}  // namespace

namespace nb {

long long launches = 0;

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

}  // namespace nb

extern "C" {

int64_t nb_weight_count(int32_t edge_dim) { return nb::WeightLayout::count(edge_dim); }
int nb_version(void) { return NB_VERSION; }
const char* nb_last_error(void) { return g_err; }
int64_t nb_launch_count(void) { return nb::launches; }
int64_t nb_buffer_count(void) { return nb::live_buffers; }

int nb_pan_create(const nb_pan_config* cfg, const float* weights, int64_t n_weights, const float* G, const float* h, nb_pan_t** out) {
  if (!cfg || !out) return fail(NB_ERR_INVALID, "null argument");
  *out = nullptr;
  if (cfg->receding < 1 || cfg->receding > 32) return fail(NB_ERR_INVALID, "receding must be in 1..32 (got %d)", cfg->receding);
  if (cfg->kinematics < 0 || cfg->kinematics > 2) return fail(NB_ERR_INVALID, "kinematics must be NB_KIN_DIFF/ACKER/OMNI");
  if (cfg->nrmp_max_num < 0 || cfg->nrmp_max_num > 32) return fail(NB_ERR_INVALID, "nrmp_max_num must be in 0..32");
  if (cfg->iter_num < 0) return fail(NB_ERR_INVALID, "iter_num must be >= 0");
  if (cfg->max_envs < 1 || cfg->max_points < 0) return fail(NB_ERR_INVALID, "max_envs >= 1 and max_points >= 0 required");
  if (!(cfg->step_time > 0)) return fail(NB_ERR_INVALID, "step_time must be positive");
  if (cfg->kinematics == NB_KIN_ACKER && !(cfg->wheelbase > 0)) return fail(NB_ERR_INVALID, "acker needs a positive wheelbase");
  if (cfg->receding * cfg->nrmp_max_num > 256)
    return fail(NB_ERR_CAPACITY, "receding * nrmp_max_num = %d exceeds 256 (the NRMP kernel keeps at most 8 hinge rows per lane)", cfg->receding * cfg->nrmp_max_num);
  const bool with_dune = cfg->nrmp_max_num > 0;
  if (with_dune) {
    if (cfg->edge_dim < 3 || cfg->edge_dim > nb::kMaxEdges) return fail(NB_ERR_INVALID, "edge_dim must be in 3..%d", nb::kMaxEdges);
    if (!weights || !G || !h) return fail(NB_ERR_INVALID, "weights, G and h are required when nrmp_max_num > 0");
    if (n_weights != nb::WeightLayout::count(cfg->edge_dim))
      return fail(NB_ERR_INVALID, "expected %d weights for edge_dim %d, got %lld", nb::WeightLayout::count(cfg->edge_dim), cfg->edge_dim, (long long)n_weights);
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(NB_ERR_NO_DEVICE, "no CUDA device available: neupan_b200 has no CPU fallback");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(NB_ERR_INVALID, "device %d out of range (%d devices)", cfg->device, ndev);
  NB_CUDA(cudaSetDevice(cfg->device));
  std::unique_ptr<nb_pan> p(new (std::nothrow) nb_pan());  // every return below but the last frees what was built
  if (!p) return fail(NB_ERR_INVALID, "out of host memory");
  p->cfg = *cfg;
  NB_CUDA(cudaDeviceGetAttribute(&p->sm_count, cudaDevAttrMultiProcessorCount, cfg->device));
  NB_CUDA(cudaDeviceGetAttribute(&p->max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, cfg->device));
  memset(&p->geo, 0, sizeof(p->geo));
  p->geo.E = cfg->edge_dim;
  const size_t B = cfg->max_envs, T1 = cfg->receding + 1, T = cfg->receding, M = cfg->nrmp_max_num, E = with_dune ? cfg->edge_dim : 1;
  if (with_dune) {
    for (int e = 0; e < cfg->edge_dim; ++e) {
      p->geo.G[e][0] = G[2 * e]; p->geo.G[e][1] = G[2 * e + 1]; p->geo.h[e] = h[e];
    }
    NB_CUDA(nb::alloc(p->d_weights, (size_t)n_weights));
    NB_CUDA(cudaMemcpy(p->d_weights.get(), weights, (size_t)n_weights * sizeof(float), cudaMemcpyHostToDevice));
    std::vector<unsigned char> image;
    p->tc_flags = nb::build_tc_image(weights, cfg->edge_dim, image, false);
    NB_CUDA(nb::alloc(p->d_tc_image, image.size()));
    NB_CUDA(cudaMemcpy(p->d_tc_image.get(), image.data(), image.size(), cudaMemcpyHostToDevice));
    nb::build_tc_image(weights, cfg->edge_dim, image, true);
    NB_CUDA(nb::alloc(p->d_tc_screen, image.size()));
    NB_CUDA(cudaMemcpy(p->d_tc_screen.get(), image.data(), image.size(), cudaMemcpyHostToDevice));
    NB_CUDA(nb::alloc(p->cand_idx, (size_t)cfg->max_envs * (cfg->receding + 1) * nb::kCandMax));
    NB_CUDA(nb::alloc(p->cand_dt, (size_t)cfg->max_envs * (cfg->receding + 1) * nb::kCandMax));
    NB_CUDA(nb::alloc(p->cand_rad, (size_t)cfg->max_envs * (cfg->receding + 1) * nb::kCandMax));
    NB_CUDA(nb::alloc(p->cand_cnt, (size_t)cfg->max_envs * (cfg->receding + 1)));
    NB_CUDA(nb::alloc(p->flag_list, (size_t)cfg->max_envs * (cfg->receding + 1)));
    NB_CUDA(nb::alloc(p->flag_count, (size_t)32));  // 4 words per internal stream: flagged items, the two refine list lengths
    NB_CUDA(nb::alloc(p->refine_list, (size_t)2 * cfg->max_envs * (cfg->receding + 1)));
    NB_CUDA(nb::alloc(p->screen_stats, (size_t)4));
    NB_CUDA(cudaMemset(p->screen_stats.get(), 0, 4 * sizeof(unsigned)));
    NB_CUDA(nb::alloc(p->coarse_stats, (size_t)2));
    NB_CUDA(cudaMemset(p->coarse_stats.get(), 0, 2 * sizeof(unsigned)));
    if (const char* e = getenv("NB_SCREEN_CMU")) { p->c_mu = (float)atof(e); p->cmu_override = true; }
  }
  NB_CUDA(nb::alloc(p->sel_mu, B * T1 * M * E));
  NB_CUDA(nb::alloc(p->sel_lam, B * T1 * M * 2));
  NB_CUDA(nb::alloc(p->sel_pts, B * T1 * M * 2));
  NB_CUDA(nb::alloc(p->sel_dist, B * T1 * M));
  NB_CUDA(nb::alloc(p->sel_count, B));
  NB_CUDA(nb::alloc(p->prev_s, B * 3 * T1));
  NB_CUDA(nb::alloc(p->prev_u, B * 2 * T));
  NB_CUDA(nb::alloc(p->prev_mu, B * T1 * M * E));
  NB_CUDA(nb::alloc(p->prev_lam, B * T1 * M * 2));
  NB_CUDA(nb::alloc(p->prev_count, B));
  NB_CUDA(nb::alloc(p->prev_valid, B));
  NB_CUDA(nb::alloc(p->active, B));
  NB_CUDA(nb::alloc(p->iters, B));
  NB_CUDA(nb::alloc(p->status, B));
  NB_CUDA(nb::alloc(p->ipm_it, B));
  NB_CUDA(cudaMemset(p->ipm_it.get(), 0, B * sizeof(int32_t)));
  NB_CUDA(nb::alloc(p->min_dist, B));
  NB_CUDA(nb::alloc(p->warm, B * nb::nrmp_warm_floats(cfg->receding, cfg->nrmp_max_num)));
  NB_CUDA(nb::alloc(p->warm_valid, B));
  NB_CUDA(nb::alloc(p->work_counters, (size_t)8));
  if (getenv("NB_NRMP_STATIC")) p->nrmp_dynamic = 0;
  if (const char* e = getenv("NB_NRMP_DEFER_STOP_MIN")) p->nrmp_defer_stop_min = atoi(e);
  if (const char* e = getenv("NB_H2D_CHUNKS")) { p->h2d_chunks = atoi(e); if (p->h2d_chunks < 1) p->h2d_chunks = 1; if (p->h2d_chunks > nb_pan::kMaxChunks) p->h2d_chunks = nb_pan::kMaxChunks; }
  if (const char* e = getenv("NB_DUNE_SKIP_T0")) p->dune_skip_t0 = atoi(e) != 0;  // developer overrides of the option defaults
  if (const char* e = getenv("NB_SCREEN_MMA")) p->screen_mma = atoi(e) != 0;
  if (const char* e = getenv("NB_SCREEN_TABLE")) p->screen_table = atoi(e) != 0;
  if (const char* e = getenv("NB_SCREEN_COARSE")) p->screen_coarse = atoi(e) != 0;
  if (const char* e = getenv("NB_NRMP_RESTART_IT")) p->warm_check_it = atoi(e);
  if (const char* e = getenv("NB_NRMP_RESTART_GAP")) p->warm_check_gap = atof(e);
  NB_CUDA(cudaMemset(p->warm_valid.get(), 0, B * sizeof(int32_t)));
  if (const char* e = getenv("NB_NRMP_GAP_TOL")) p->nrmp_gap_tol = atof(e);
  NB_CUDA(cudaMemset(p->prev_valid.get(), 0, B * sizeof(int32_t)));
  NB_CUDA(cudaMemset(p->prev_count.get(), 0, B * sizeof(int32_t)));
  NB_CUDA(cudaMemset(p->sel_count.get(), 0, B * sizeof(int32_t)));
  // the default: two sub-batches on internal streams (streams / events are made here)
  if (int rc = nb_pan_set_option(p.get(), NB_OPT_OVERLAP, 2)) return rc;
  *out = p.release();
  return NB_OK;
}

int nb_pan_destroy(nb_pan_t* p) {
  if (!p) return NB_OK;
  cudaSetDevice(p->cfg.device);
  delete p;
  return NB_OK;
}

int nb_pan_set_adjust(nb_pan_t* p, const float q_s[3], float p_u, float eta, float d_max, float d_min) {
  if (!p || !q_s) return fail(NB_ERR_INVALID, "null argument");
  for (int i = 0; i < 3; ++i) p->cfg.q_s[i] = q_s[i];
  p->cfg.p_u = p_u; p->cfg.eta = eta; p->cfg.d_max = d_max; p->cfg.d_min = d_min;
  return NB_OK;
}

int nb_pan_set_iteration(nb_pan_t* p, int32_t iter_num, float iter_threshold) {
  if (!p || iter_num < 0) return fail(NB_ERR_INVALID, "bad argument");
  p->cfg.iter_num = iter_num; p->cfg.iter_threshold = iter_threshold;
  return NB_OK;
}

int nb_pan_set_option(nb_pan_t* p, int32_t option, int32_t value) {
  if (!p) return fail(NB_ERR_INVALID, "null handle");
  if (option == NB_OPT_DUNE_KERNEL) {
    if (value != 2 && value != 4)
      return fail(NB_ERR_INVALID, "NB_OPT_DUNE_KERNEL takes 2 (wgmma on every point) or 4 (wgmma with screening), got %d", value);
    p->dune_variant = value;
    if (value == 4 && p->d_tc_screen) {
      NB_CUDA(cudaSetDevice(p->cfg.device));
      if (!p->screen_calibrated)
        if (int rc = calibrate_screen(p, nullptr)) return rc;
      if (p->screen_table && !p->tab_built) return build_screen_table(p);
    }
    return NB_OK;
  }
  if (option == NB_OPT_DUNE_SCREEN_TABLE) {
    if (value < 0 || value > 1) return fail(NB_ERR_INVALID, "NB_OPT_DUNE_SCREEN_TABLE takes 0 or 1");
    p->screen_table = value;
    if (value == 1 && p->dune_variant == 4 && p->d_tc_screen && !p->tab_built) {
      NB_CUDA(cudaSetDevice(p->cfg.device));
      return build_screen_table(p);
    }
    return NB_OK;
  }
  if (option == NB_OPT_OVERLAP) {
    if (value < 1 || value > 4) return fail(NB_ERR_INVALID, "NB_OPT_OVERLAP takes 1..4");
    NB_CUDA(cudaSetDevice(p->cfg.device));
    for (int i = 0; i < value && value > 1; ++i) {
      if (!p->streams[i]) NB_CUDA(nb::create(p->streams[i]));
      if (!p->ev_join[i]) NB_CUDA(nb::create(p->ev_join[i]));
    }
    if (value > 1 && !p->ev_fork) NB_CUDA(nb::create(p->ev_fork));
    p->overlap = value;
    return NB_OK;
  }
  if (option == NB_OPT_DIFFERENTIABLE) {
    if (value < 0 || value > 1) return fail(NB_ERR_INVALID, "NB_OPT_DIFFERENTIABLE takes 0 or 1");
    p->differentiable = value;
    return NB_OK;
  }
  if (option == NB_OPT_DUNE_SCREEN_MMA || option == NB_OPT_DUNE_SKIP_T0) {
    if (value < 0 || value > 1) return fail(NB_ERR_INVALID, "NB_OPT_DUNE_SCREEN_MMA / NB_OPT_DUNE_SKIP_T0 take 0 or 1");
    (option == NB_OPT_DUNE_SCREEN_MMA ? p->screen_mma : p->dune_skip_t0) = value;
    return NB_OK;
  }
  if (option == NB_OPT_NRMP_WARM) {
    if (value < 0 || value > 1) return fail(NB_ERR_INVALID, "NB_OPT_NRMP_WARM takes 0 or 1");
    p->nrmp_warm = value;
    return NB_OK;
  }
  return fail(NB_ERR_INVALID, "unknown option %d", option);
}

int nb_pan_reset_state_async(nb_pan_t* p, void* stream) {
  if (!p) return fail(NB_ERR_INVALID, "null handle");
  NB_CUDA(cudaSetDevice(p->cfg.device));
  NB_CUDA(cudaMemsetAsync(p->prev_valid.get(), 0, (size_t)p->cfg.max_envs * sizeof(int32_t), (cudaStream_t)stream));
  NB_CUDA(cudaMemsetAsync(p->prev_count.get(), 0, (size_t)p->cfg.max_envs * sizeof(int32_t), (cudaStream_t)stream));
  return NB_OK;
}

int nb_pan_reset_envs_async(nb_pan_t* p, int32_t B, const int32_t* mask, void* stream) {
  if (!p || !mask) return fail(NB_ERR_INVALID, "nb_pan_reset_envs_async: null argument");
  if (B < 1 || B > p->cfg.max_envs) return fail(NB_ERR_CAPACITY, "B = %d outside [1, max_envs = %d]", B, p->cfg.max_envs);
  NB_CUDA(cudaSetDevice(p->cfg.device));
  reset_envs_kernel<<<(B + 255) / 256, 256, 0, (cudaStream_t)stream>>>(B, mask, p->prev_valid.get(), p->prev_count.get());
  ++nb::launches;
  NB_CUDA(cudaGetLastError());
  return NB_OK;
}

int nb_pan_reset_state(nb_pan_t* p) {
  if (int rc = nb_pan_reset_state_async(p, nullptr)) return rc;
  NB_CUDA(cudaStreamSynchronize(nullptr));
  return NB_OK;
}

int nb_dune_forward(nb_pan_t* p, int32_t B, int32_t N, const float* nom_s, const float* points, const float* velocities,
                    const int32_t* num_points, float* out_min_distance, void* stream) {
  if (int rc = check_forward_args(p, B, N)) return rc;
  if (p->cfg.nrmp_max_num == 0) return fail(NB_ERR_INVALID, "handle was created in no_obs mode");
  if (!nom_s || !points) return fail(NB_ERR_INVALID, "nom_s and points are required");
  if (N == 0) return fail(NB_ERR_INVALID, "N must be positive");
  NB_CUDA(cudaSetDevice(p->cfg.device));
  nb::DuneParams prm = dune_params(p);
  prm.nom_s = nom_s; prm.points = points; prm.velocities = velocities; prm.num_points = num_points;
  prm.min_dist = out_min_distance;
  prm.B = B; prm.N = N;
  set_screen_table(p, prm);
  return nb::launch_dune_tc(prm, p->d_tc_image.get(), p->d_tc_screen.get(), p->tc_flags, p->dune_variant == 4, p->sm_count, p->max_smem_optin,
                            (cudaStream_t)stream);
}

int nb_nrmp_forward(nb_pan_t* p, int32_t B, const float* nom_s, const float* nom_u, const float* ref_s, const float* ref_us,
                    const float* fa, const float* fb, float* out_s, float* out_u, float* out_d, int32_t* out_status, void* stream) {
  if (int rc = check_forward_args(p, B, 0)) return rc;
  if (!nom_s || !nom_u || !ref_s || !ref_us || !out_s || !out_u || !out_d) return fail(NB_ERR_INVALID, "null tensor argument");
  if ((fa == nullptr) != (fb == nullptr)) return fail(NB_ERR_INVALID, "fa and fb must be given together");
  NB_CUDA(cudaSetDevice(p->cfg.device));
  nb::NrmpParams prm = nrmp_params(p);
  prm.nom_s = nom_s; prm.nom_u = nom_u; prm.ref_s = ref_s; prm.ref_us = ref_us; prm.fa = fa; prm.fb = fb;
  prm.out_s = out_s; prm.out_u = out_u; prm.out_d = out_d; prm.status = out_status;
  prm.ipm_iters = p->ipm_it.get();  // nb_pan_read_diagnostics
  prm.B = B;
  return nb::launch_nrmp(prm, nrmp_launch(p, 0), (cudaStream_t)stream);
}

namespace {
// env chunks whose inputs arrive on another stream: chunk c = environments [bound[c], bound[c+1]), usable once ev[c] has fired
struct ChunkPlan {
  int n = 0;
  int bound[nb_pan::kMaxChunks + 1] = {};
  cudaEvent_t ev[nb_pan::kMaxChunks] = {};
};
int pan_forward_impl(nb_pan_t* p, int32_t B, int32_t N, const float* nom_s, const float* nom_u, const float* ref_s, const float* ref_us,
                     const float* points, const float* velocities, const int32_t* num_points, float* out_s, float* out_u, float* out_d,
                     float* out_min_distance, int32_t* out_iters, int32_t* out_status, void* stream, const ChunkPlan* plan);
}  // namespace

int nb_pan_forward(nb_pan_t* p, int32_t B, int32_t N, const float* nom_s, const float* nom_u, const float* ref_s, const float* ref_us,
                   const float* points, const float* velocities, const int32_t* num_points, float* out_s, float* out_u, float* out_d,
                   float* out_min_distance, int32_t* out_iters, int32_t* out_status, void* stream) {
  return pan_forward_impl(p, B, N, nom_s, nom_u, ref_s, ref_us, points, velocities, num_points, out_s, out_u, out_d, out_min_distance, out_iters,
                          out_status, stream, nullptr);
}

namespace {
int pan_forward_impl(nb_pan_t* p, int32_t B, int32_t N, const float* nom_s, const float* nom_u, const float* ref_s, const float* ref_us,
                     const float* points, const float* velocities, const int32_t* num_points, float* out_s, float* out_u, float* out_d,
                     float* out_min_distance, int32_t* out_iters, int32_t* out_status, void* stream, const ChunkPlan* plan) {
  if (int rc = check_forward_args(p, B, N)) return rc;
  if (!nom_s || !nom_u || !ref_s || !ref_us || !out_s || !out_u || !out_d) return fail(NB_ERR_INVALID, "null tensor argument");
  if (velocities && !points) return fail(NB_ERR_INVALID, "velocities given without points");
  NB_CUDA(cudaSetDevice(p->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const nb_pan_config& c = p->cfg;
  const int T = c.receding, T1 = T + 1;
  const bool with_dune = c.nrmp_max_num > 0 && points != nullptr && N > 0;  // pan.py:130
  if (p->differentiable && (!p->adj.rec || p->adj.iters < c.iter_num)) {  // (re)allocate the adjoint records for K iterations
    p->adj = {};  // the old set goes first; a failure below leaves none, never part of one
    const size_t Bm = c.max_envs, Ks = c.iter_num > 0 ? c.iter_num : 1;
    nb_pan::Adjoint a;
    NB_CUDA(nb::alloc(a.rec, Ks * Bm * nb::nrmp_adj_doubles(T, c.nrmp_max_num)));
    NB_CUDA(nb::alloc(a.valid, Ks * Bm));
    NB_CUDA(nb::alloc(a.gs, Bm * 3 * T1));
    NB_CUDA(nb::alloc(a.gu, Bm * 2 * T));
    NB_CUDA(nb::alloc(a.gd, Bm * T));
    NB_CUDA(nb::alloc(a.gtheta, Bm * 7));
    a.iters = (int)Ks;
    p->adj = std::move(a);
  }
  if (p->differentiable) NB_CUDA(cudaMemsetAsync(p->adj.valid.get(), 0, (size_t)p->adj.iters * c.max_envs * sizeof(int32_t), st));
  if (plan && plan->n > 0) NB_CUDA(cudaStreamWaitEvent(st, plan->ev[0], 0));  // the small tensors travel ahead of chunk 0
  const int tb = 128, gb = (B + tb - 1) / tb;
  init_run_kernel<<<gb, tb, 0, st>>>(B, p->active.get(), p->iters.get(), p->status.get(), p->min_dist.get(), p->sel_count.get(), p->warm_valid.get());
  ++nb::launches;
  // the nominal trajectory lives in the output buffers and is updated in place every iteration
  NB_CUDA(cudaMemcpyAsync(out_s, nom_s, (size_t)B * 3 * T1 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  NB_CUDA(cudaMemcpyAsync(out_u, nom_u, (size_t)B * 2 * T * sizeof(float), cudaMemcpyDeviceToDevice, st));
  NB_CUDA(cudaMemsetAsync(out_d, 0, (size_t)B * T * sizeof(float), st));
  // K iterations of {DUNE, NRMP} for the environments [lo, hi) on stream s
  auto run_range = [&](int lo, int hi, cudaStream_t s, int counter_slot, int k0, int k1) -> int {
    const int nb_ = hi - lo;
    const size_t T1s = (size_t)T1, Ms = (size_t)c.nrmp_max_num, Es = (size_t)(c.edge_dim > 0 ? c.edge_dim : 1);
    const bool screen = p->dune_variant == 4;
    auto dune = [&](const nb::DuneParams& d) {
      return nb::launch_dune_tc(d, p->d_tc_image.get(), p->d_tc_screen.get(), p->tc_flags, screen, p->sm_count, p->max_smem_optin, s);
    };
    nb::DuneParams d{};  // the environments [lo, hi)
    if (with_dune) {
      d = dune_params(p);
      d.nom_s = out_s; d.points = points; d.velocities = velocities; d.num_points = num_points;
      d.active = p->active.get(); d.min_dist = p->min_dist.get();
      d.B = nb_; d.N = N;
      d.flag_count += 4 * counter_slot;
      set_screen_table(p, d);
      dune_offset(d, (size_t)lo);
    }
    for (int k = k0; k < k1; ++k) {
      if (with_dune) {
        d.skip_t0 = (k > 0 && p->dune_skip_t0) ? 1 : 0;  // the step-0 items of iteration 0 stand (DuneParams::skip_t0)
        if (k == 0 && plan && plan->n > 1) {
          // the first DUNE pass of this range chunk by chunk, each as soon as its points have landed: the upload of chunk c+1 overlaps the
          // work on chunk c (d describes the environments [lo, hi); a chunk's part of them is [clo, chi))
          for (int ch = 0; ch < plan->n; ++ch) {
            const int clo = plan->bound[ch] > lo ? plan->bound[ch] : lo, chi = plan->bound[ch + 1] < hi ? plan->bound[ch + 1] : hi;
            if (chi <= clo) continue;
            NB_CUDA(cudaStreamWaitEvent(s, plan->ev[ch], 0));
            nb::DuneParams dc = d;
            dune_offset(dc, (size_t)(clo - lo));
            dc.B = chi - clo;
            if (int rc = dune(dc)) return rc;
          }
        } else {
          if (int rc = dune(d)) return rc;
        }
      }
      nb::NrmpParams n = nrmp_params(p);
      n.nom_s = out_s + (size_t)lo * 3 * T1s; n.nom_u = out_u + (size_t)lo * 2 * T; n.ref_s = ref_s + (size_t)lo * 3 * T1s; n.ref_us = ref_us + (size_t)lo * T;
      if (with_dune) { n.sel_mu = d.sel_mu; n.sel_lam = d.sel_lam; n.sel_pts = d.sel_pts; n.sel_count = d.sel_count; }
      n.out_s = out_s + (size_t)lo * 3 * T1s; n.out_u = out_u + (size_t)lo * 2 * T; n.out_d = out_d + (size_t)lo * T;
      n.status = p->status.get() + lo; n.iters = p->iters.get() + lo; n.active = p->active.get() + lo; n.ipm_iters = p->ipm_it.get() + lo;
      n.prev_s = p->prev_s.get() + (size_t)lo * 3 * T1s; n.prev_u = p->prev_u.get() + (size_t)lo * 2 * T;
      n.prev_mu = p->prev_mu.get() + (size_t)lo * T1s * Ms * Es; n.prev_lam = p->prev_lam.get() + (size_t)lo * T1s * Ms * 2;
      n.prev_count = p->prev_count.get() + lo; n.prev_valid = p->prev_valid.get() + lo;
      if (p->differentiable && p->adj.rec && k < p->adj.iters) {
        n.adj_save = p->adj.rec.get() + ((size_t)k * c.max_envs + lo) * nb::nrmp_adj_doubles(T, c.nrmp_max_num);
        n.adj_valid = p->adj.valid.get() + (size_t)k * c.max_envs + lo;
      }
      if (p->nrmp_warm) {
        n.warm = p->warm.get() + (size_t)lo * nb::nrmp_warm_floats(T, c.nrmp_max_num);
        n.warm_valid = p->warm_valid.get() + lo;
      }
      n.B = nb_;
      if (int rc = nb::launch_nrmp(n, nrmp_launch(p, counter_slot), s)) return rc;
    }
    return NB_OK;
  };
  const int parts = (p->overlap > 1 && with_dune && B >= 64 * p->overlap) ? p->overlap : 1;
  if (parts == 1) {
    if (int rc = run_range(0, B, st, 0, 0, c.iter_num)) return rc;
  } else {
    // sub-batches on internal streams: the DUNE kernel of one part (issue / tensor / MUFU bound) shares the SMs with the
    // NRMP kernel of another (latency bound, few warps)
    NB_CUDA(cudaEventRecord(p->ev_fork.get(), st));
    for (int i = 0; i < parts; ++i) NB_CUDA(cudaStreamWaitEvent(p->streams[i].get(), p->ev_fork.get(), 0));
    // enqueue order: iteration by iteration, alternating the streams (every sub-batch starts at once; NB_PAN_INTERLEAVE=0, a developer
    // switch, enqueues all K iterations of one sub-batch before the next)
    static int interleave = -1;
    if (interleave < 0) {
      const char* v = getenv("NB_PAN_INTERLEAVE");
      interleave = v ? atoi(v) : 1;
    }
    auto range_of = [&](int i, int& lo, int& hi) { lo = (int)((long long)B * i / parts); hi = (int)((long long)B * (i + 1) / parts); };
    if (interleave) {
      for (int k = 0; k < c.iter_num; ++k)
        for (int i = 0; i < parts; ++i) {
          int lo, hi;
          range_of(i, lo, hi);
          if (int rc = run_range(lo, hi, p->streams[i].get(), 1 + i, k, k + 1)) return rc;
        }
    } else {
      for (int i = 0; i < parts; ++i) {
        int lo, hi;
        range_of(i, lo, hi);
        if (int rc = run_range(lo, hi, p->streams[i].get(), 1 + i, 0, c.iter_num)) return rc;
      }
    }
    for (int i = 0; i < parts; ++i) {
      NB_CUDA(cudaEventRecord(p->ev_join[i].get(), p->streams[i].get()));
      NB_CUDA(cudaStreamWaitEvent(st, p->ev_join[i].get(), 0));
    }
  }
  finish_run_kernel<<<gb, tb, 0, st>>>(B, p->iters.get(), p->status.get(), p->min_dist.get(), out_iters, out_status, out_min_distance);
  ++nb::launches;
  NB_CUDA(cudaGetLastError());
  return NB_OK;
}
}  // namespace

int nb_pan_backward(nb_pan_t* p, int32_t B, const float* ref_s, const float* ref_us, const float* grad_s, const float* grad_u, const float* grad_d,
                    float* grad_theta, void* stream) {
  if (int rc = check_forward_args(p, B, 0)) return rc;
  if (!p->differentiable || !p->adj.rec) return fail(NB_ERR_INVALID, "nb_pan_backward needs a forward in differentiable mode (NB_OPT_DIFFERENTIABLE = 1) first");
  if (!ref_s || !ref_us || !grad_theta) return fail(NB_ERR_INVALID, "null tensor argument");
  NB_CUDA(cudaSetDevice(p->cfg.device));
  const nb_pan_config& c = p->cfg;
  nb::NrmpAdjParams a{};
  a.rec = p->adj.rec.get(); a.rec_valid = p->adj.valid.get();
  a.iters = p->iters.get(); a.ref_s = ref_s; a.ref_us = ref_us;
  a.g_s = p->adj.gs.get(); a.g_u = p->adj.gu.get(); a.g_d = p->adj.gd.get(); a.grad_theta = p->adj.gtheta.get();
  a.B = B; a.T = c.receding; a.M = c.nrmp_max_num; a.kin = c.kinematics;
  for (int i = 0; i < 3; ++i) a.q[i] = c.q_s[i];
  a.p_u = c.p_u; a.d_min = c.d_min; a.bk = c.bk;
  const int K = c.iter_num < p->adj.iters ? c.iter_num : p->adj.iters;
  return nb::launch_nrmp_backward(a, K, c.max_envs, grad_s, grad_u, grad_d, grad_theta, (cudaStream_t)stream);
}

int nb_pan_read_selection(nb_pan_t* p, int32_t B, float* sel_mu, float* sel_lam, float* sel_points, float* sel_distance,
                          int32_t* sel_count, void* stream) {
  if (int rc = check_forward_args(p, B, 0)) return rc;
  NB_CUDA(cudaSetDevice(p->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t T1 = p->cfg.receding + 1, M = p->cfg.nrmp_max_num, E = p->cfg.edge_dim;
  if (sel_mu) NB_CUDA(cudaMemcpyAsync(sel_mu, p->sel_mu.get(), (size_t)B * T1 * M * E * 4, cudaMemcpyDeviceToDevice, st));
  if (sel_lam) NB_CUDA(cudaMemcpyAsync(sel_lam, p->sel_lam.get(), (size_t)B * T1 * M * 2 * 4, cudaMemcpyDeviceToDevice, st));
  if (sel_points) NB_CUDA(cudaMemcpyAsync(sel_points, p->sel_pts.get(), (size_t)B * T1 * M * 2 * 4, cudaMemcpyDeviceToDevice, st));
  if (sel_distance) NB_CUDA(cudaMemcpyAsync(sel_distance, p->sel_dist.get(), (size_t)B * T1 * M * 4, cudaMemcpyDeviceToDevice, st));
  if (sel_count) NB_CUDA(cudaMemcpyAsync(sel_count, p->sel_count.get(), (size_t)B * 4, cudaMemcpyDeviceToDevice, st));
  return NB_OK;
}

int nb_pan_read_screen_stats(nb_pan_t* p, float* max_error_ratio, int32_t* counts, int32_t reset) {
  if (!p || !max_error_ratio || !counts) return fail(NB_ERR_INVALID, "nb_pan_read_screen_stats: null argument");
  if (!p->screen_stats) return fail(NB_ERR_INVALID, "handle was created in no_obs mode");
  NB_CUDA(cudaSetDevice(p->cfg.device));
  NB_CUDA(cudaDeviceSynchronize());
  unsigned h[4];
  NB_CUDA(cudaMemcpy(h, p->screen_stats.get(), sizeof(h), cudaMemcpyDeviceToHost));
  memcpy(max_error_ratio, &h[0], 4);
  max_error_ratio[1] = p->c_mu;
  max_error_ratio[2] = p->screen_cal_ratio;
  counts[0] = (int32_t)h[1]; counts[1] = (int32_t)h[2]; counts[2] = (int32_t)h[3];
  if (reset) NB_CUDA(cudaMemset(p->screen_stats.get(), 0, sizeof(h)));
  return NB_OK;
}

int nb_pan_read_screen_coarse(nb_pan_t* p, int32_t* counts, int32_t reset) {
  if (!p || !counts) return fail(NB_ERR_INVALID, "nb_pan_read_screen_coarse: null argument");
  if (!p->coarse_stats) return fail(NB_ERR_INVALID, "handle was created in no_obs mode");
  NB_CUDA(cudaSetDevice(p->cfg.device));
  NB_CUDA(cudaDeviceSynchronize());
  unsigned h[2];
  NB_CUDA(cudaMemcpy(h, p->coarse_stats.get(), sizeof(h), cudaMemcpyDeviceToHost));
  counts[0] = (int32_t)h[0]; counts[1] = (int32_t)h[1];
  if (reset) NB_CUDA(cudaMemset(p->coarse_stats.get(), 0, sizeof(h)));
  return NB_OK;
}

int nb_pan_read_screen_table(nb_pan_t* p, float* info) {
  if (!p || !info) return fail(NB_ERR_INVALID, "nb_pan_read_screen_table: null argument");
  info[0] = p->tab_h;
  info[1] = p->tab_half;
  info[2] = p->tab_cell ? (float)((double)p->tab_n * p->tab_n * (sizeof(float4) + sizeof(float)) + (double)p->tab_cn * p->tab_cn * sizeof(uint32_t)) : 0.f;
  info[3] = p->tab_ms;
  info[4] = p->tab_ratio;
  return NB_OK;
}

int nb_pan_read_diagnostics(nb_pan_t* p, int32_t B, int32_t* ipm_iterations, void* stream) {
  if (int rc = check_forward_args(p, B, 0)) return rc;
  NB_CUDA(cudaSetDevice(p->cfg.device));
  if (ipm_iterations) NB_CUDA(cudaMemcpyAsync(ipm_iterations, p->ipm_it.get(), (size_t)B * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return NB_OK;
}

namespace {
// Upload of the host inputs into the handle's staging buffer on the copy stream, in env chunks, and the forward pass on `st` that
// consumes them chunk by chunk; outputs go to the device pointers given.  Nothing is synchronised here.
int pan_forward_from_host(nb_pan_t* p, int32_t B, int32_t N, const float* nom_s, const float* nom_u, const float* ref_s, const float* ref_us,
                          const float* points, const float* velocities, const int32_t* num_points, float* out_s, float* out_u, float* out_d,
                          float* out_min_distance, int32_t* out_iters, int32_t* out_status, cudaStream_t st) {
  const size_t T = p->cfg.receding, T1 = T + 1;
  const size_t n_s = (size_t)B * 3 * T1, n_u = (size_t)B * 2 * T, n_r = (size_t)B * T, n_p = (size_t)B * 2 * N;
  const size_t in_floats = 2 * n_s + n_u + n_r + 2 * n_p;
  if (!p->copy_stream) NB_CUDA(nb::create(p->copy_stream));
  if (!p->ev_inputs_free) NB_CUDA(nb::create(p->ev_inputs_free));
  for (nb::Event& ev : p->ev_chunk)
    if (!ev) NB_CUDA(nb::create(ev));
  cudaStream_t cs = p->copy_stream.get();
  // whatever `st` still does with the staging buffer (the previous call) must be over before it is overwritten
  NB_CUDA(cudaEventRecord(p->ev_inputs_free.get(), st));
  NB_CUDA(cudaStreamWaitEvent(cs, p->ev_inputs_free.get(), 0));
  if (in_floats > p->h_in_floats) {
    NB_CUDA(cudaStreamSynchronize(cs));
    p->h_in_floats = 0;
    NB_CUDA(nb::alloc(p->h_in, in_floats));
    p->h_in_floats = in_floats;
  }
  if (!p->h_np) NB_CUDA(nb::alloc(p->h_np, (size_t)p->cfg.max_envs));
  float* d = p->h_in.get();
  float* d_nom_s = d; d += n_s;
  float* d_ref_s = d; d += n_s;
  float* d_nom_u = d; d += n_u;
  float* d_ref_us = d; d += n_r;
  float* d_pts = d; d += n_p;
  float* d_vel = d;
  auto h2d = [&](void* dst, const void* src, size_t bytes) { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, cs); };
  NB_CUDA(h2d(d_nom_s, nom_s, n_s * 4));
  NB_CUDA(h2d(d_ref_s, ref_s, n_s * 4));
  NB_CUDA(h2d(d_nom_u, nom_u, n_u * 4));
  NB_CUDA(h2d(d_ref_us, ref_us, n_r * 4));
  if (num_points) NB_CUDA(h2d(p->h_np.get(), num_points, (size_t)B * 4));
  const bool with_pts = points && N > 0;
  ChunkPlan plan;
  plan.n = (with_pts && B >= 64 * p->h2d_chunks) ? p->h2d_chunks : 1;
  if (with_pts && p->overlap > 1 && B >= 64 * p->overlap) {  // sub-batches on internal streams: chunk boundaries that contain theirs
    plan.n = p->overlap * (B >= 128 * p->overlap ? 2 : 1);
    if (plan.n > nb_pan::kMaxChunks) plan.n = p->overlap;
  }
  for (int c = 0; c <= plan.n; ++c) plan.bound[c] = (int)((long long)B * c / plan.n);
  for (int c = 0; c < plan.n; ++c) {
    const size_t lo = (size_t)plan.bound[c] * 2 * N, cnt = (size_t)(plan.bound[c + 1] - plan.bound[c]) * 2 * N;
    if (with_pts && cnt) NB_CUDA(h2d(d_pts + lo, points + lo, cnt * 4));
    if (with_pts && velocities && cnt) NB_CUDA(h2d(d_vel + lo, velocities + lo, cnt * 4));
    plan.ev[c] = p->ev_chunk[c].get();
    NB_CUDA(cudaEventRecord(plan.ev[c], cs));
  }
  return pan_forward_impl(p, B, N, d_nom_s, d_nom_u, d_ref_s, d_ref_us, with_pts ? d_pts : nullptr, (with_pts && velocities) ? d_vel : nullptr,
                          num_points ? p->h_np.get() : nullptr, out_s, out_u, out_d, out_min_distance, out_iters, out_status, st, &plan);
}
}  // namespace

int nb_pan_forward_h2d(nb_pan_t* p, int32_t B, int32_t N, const float* nom_s, const float* nom_u, const float* ref_s, const float* ref_us,
                       const float* points, const float* velocities, const int32_t* num_points, float* out_s, float* out_u, float* out_d,
                       float* out_min_distance, int32_t* out_iters, int32_t* out_status, void* stream) {
  if (int rc = check_forward_args(p, B, N)) return rc;
  if (!nom_s || !nom_u || !ref_s || !ref_us || !out_s || !out_u || !out_d) return fail(NB_ERR_INVALID, "null tensor argument");
  NB_CUDA(cudaSetDevice(p->cfg.device));
  return pan_forward_from_host(p, B, N, nom_s, nom_u, ref_s, ref_us, points, velocities, num_points, out_s, out_u, out_d, out_min_distance, out_iters,
                               out_status, (cudaStream_t)stream);
}

int nb_pan_forward_host(nb_pan_t* p, int32_t B, int32_t N, const float* nom_s, const float* nom_u, const float* ref_s,
                        const float* ref_us, const float* points, const float* velocities, const int32_t* num_points, float* out_s,
                        float* out_u, float* out_d, float* out_min_distance, int32_t* out_iters, int32_t* out_status, void* stream) {
  if (int rc = check_forward_args(p, B, N)) return rc;
  if (!nom_s || !nom_u || !ref_s || !ref_us || !out_s || !out_u || !out_d) return fail(NB_ERR_INVALID, "null tensor argument");
  NB_CUDA(cudaSetDevice(p->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t T = p->cfg.receding, T1 = T + 1;
  const size_t n_s = (size_t)B * 3 * T1, n_u = (size_t)B * 2 * T, n_r = (size_t)B * T;
  const size_t out_floats = n_s + n_u + n_r + (size_t)B;
  if (out_floats > p->h_out_floats) {
    p->h_out_floats = 0;
    NB_CUDA(nb::alloc(p->h_out, out_floats));
    p->h_out_floats = out_floats;
  }
  if (!p->h_io) NB_CUDA(nb::alloc(p->h_io, 2 * (size_t)p->cfg.max_envs));
  int32_t* io = p->h_io.get();
  float* o = p->h_out.get();
  float* o_s = o; o += n_s;
  float* o_u = o; o += n_u;
  float* o_d = o; o += n_r;
  float* o_md = o;
  int rc = pan_forward_from_host(p, B, N, nom_s, nom_u, ref_s, ref_us, points, velocities, num_points, o_s, o_u, o_d, o_md, io,
                                 io + p->cfg.max_envs, st);
  if (rc) return rc;
  auto d2h = [&](void* dst, const void* src, size_t bytes) { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st); };
  NB_CUDA(d2h(out_s, o_s, n_s * 4));
  NB_CUDA(d2h(out_u, o_u, n_u * 4));
  NB_CUDA(d2h(out_d, o_d, n_r * 4));
  if (out_min_distance) NB_CUDA(d2h(out_min_distance, o_md, (size_t)B * 4));
  if (out_iters) NB_CUDA(d2h(out_iters, io, (size_t)B * 4));
  if (out_status) NB_CUDA(d2h(out_status, io + p->cfg.max_envs, (size_t)B * 4));
  NB_CUDA(cudaStreamSynchronize(st));
  return NB_OK;
}

}  // extern "C"
