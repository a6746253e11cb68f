// C ABI of the single-kernel entry points (include/neupan_b200.h): lidar scans to points, the initial path handle, and the labels and
// training of DUNE.
#include <cstdlib>
#include <memory>
#include <new>

#include "host_common.h"
#include "scan_kernel.cuh"
#include "ipath_kernel.cuh"
#include "dune_train_kernel.cuh"

using nb::fail;

struct nb_ipath {
  nb_ipath_config cfg;
  int B = 0;
  int64_t P = 0;
  nb::DeviceArray<double> d_pts;
  nb::DeviceArray<int32_t> d_curve_begin;
  nb::DeviceArray<int32_t> d_env_curve_begin;
  nb::DeviceArray<double> d_interval;
  nb::DeviceArray<int32_t> d_curve_index;
  nb::DeviceArray<int32_t> d_point_index;
  nb::DeviceArray<int32_t> d_arrive_flag;
};

struct nb_dune_train {
  int E = 0, device = 0, n_weights = 0;
  float G[nb::kMaxEdges][2];
  float h[nb::kMaxEdges];
  nb::DeviceArray<float> d_weights, d_m, d_v, d_thetas;
  nb::DeviceArray<double> d_losses;
  size_t thetas_cap = 0;
  long long steps = 0;  // optimiser steps taken so far (Adam bias correction)
};

extern "C" {

int nb_scan_to_points(int32_t B, int32_t R, const float* ranges, const float* velocity, const double* states,
                      const nb_scan_config* cfg, int32_t max_points, float* points, float* velocities_out,
                      int32_t* counts, void* stream) {
  if (!cfg || !ranges || !states || !points || !counts) return fail(NB_ERR_INVALID, "nb_scan_to_points: null argument");
  if (B < 0 || R < 1 || max_points < 1) return fail(NB_ERR_INVALID, "nb_scan_to_points: B=%d R=%d max_points=%d", B, R, max_points);
  if (cfg->down_sample < 1) return fail(NB_ERR_INVALID, "down_sample must be >= 1 (got %d)", cfg->down_sample);
  if ((size_t)R * sizeof(int32_t) > 200 * 1024) return fail(NB_ERR_CAPACITY, "R=%d beams exceed the shared-memory list (51200)", R);
  if (B == 0) return NB_OK;
  nb::ScanParams prm;
  prm.B = B; prm.R = R; prm.max_points = max_points;
  prm.ranges = ranges; prm.velocity = velocity; prm.states = states;
  prm.angle_min = cfg->angle_min; prm.angle_max = cfg->angle_max; prm.range_min = cfg->range_min; prm.range_max = cfg->range_max;
  prm.off_x = cfg->scan_offset[0]; prm.off_y = cfg->scan_offset[1]; prm.off_th = cfg->scan_offset[2];
  prm.angle_lo = cfg->angle_range[0]; prm.angle_hi = cfg->angle_range[1];
  prm.down_sample = cfg->down_sample; prm.velocity_mode = cfg->velocity_mode ? 1 : 0;
  prm.points = points; prm.vel_out = velocities_out; prm.counts = counts;
  const size_t smem = (size_t)R * sizeof(int32_t);
  static const bool generic_only = getenv("NB_SCAN_GENERIC") != nullptr;  // developer switch: force the chunked kernel
  if (R <= nb::kScanMaxChunks * 1024 && !generic_only) {  // all ranges of a thread in registers, one barrier
    int threads = 128;
    while (threads * nb::kScanMaxChunks < R) threads *= 2;
    if (R >= 512 && threads < 256) threads = 256;
    nb::scan_to_points_fast_kernel<<<B, threads, smem, (cudaStream_t)stream>>>(prm);
  } else {
    if (smem > 48 * 1024) NB_CUDA(cudaFuncSetAttribute(nb::scan_to_points_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    nb::scan_to_points_kernel<<<B, 256, smem, (cudaStream_t)stream>>>(prm);
  }
  ++nb::launches;
  NB_CUDA(cudaGetLastError());
  return NB_OK;
}

// ---- DUNE training (SURVEY 8f row 4) -------------------------------------------------------------------------------
int nb_dune_labels(int32_t E, const float* G, const float* h, int64_t n, const double* points, float* points_f32, float* mu, float* dist, void* stream) {
  if (E < 3 || E > nb::kMaxEdges || !G || !h) return fail(NB_ERR_INVALID, "nb_dune_labels: edge_dim must be in 3..%d and G, h given", nb::kMaxEdges);
  if (n < 0 || (n > 0 && (!points || !points_f32 || !mu || !dist))) return fail(NB_ERR_INVALID, "nb_dune_labels: null argument");
  if (n == 0) return NB_OK;
  nb::DuneLabelParams prm;
  prm.n = (int)n; prm.E = E;
  for (int e = 0; e < E; ++e) { prm.G[e][0] = G[2 * e]; prm.G[e][1] = G[2 * e + 1]; prm.h[e] = h[e]; }
  prm.points = points; prm.points_f32 = points_f32; prm.mu = mu; prm.dist = dist;
  nb::dune_label_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(prm);
  ++nb::launches;
  NB_CUDA(cudaGetLastError());
  return NB_OK;
}

int nb_dune_train_create(int32_t E, const float* G, const float* h, const float* weights, int64_t n_weights, int32_t device, nb_dune_train_t** out) {
  if (!out || !G || !h || !weights) return fail(NB_ERR_INVALID, "nb_dune_train_create: null argument");
  *out = nullptr;
  if (E < 3 || E > nb::kMaxEdges) return fail(NB_ERR_INVALID, "edge_dim must be in 3..%d", nb::kMaxEdges);
  if (n_weights != nb::WeightLayout::count(E)) return fail(NB_ERR_INVALID, "expected %d weights for edge_dim %d", nb::WeightLayout::count(E), E);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || device < 0 || device >= ndev)
    return fail(NB_ERR_NO_DEVICE, "no CUDA device available: neupan_b200 has no CPU fallback");
  NB_CUDA(cudaSetDevice(device));
  std::unique_ptr<nb_dune_train> t(new (std::nothrow) nb_dune_train());
  if (!t) return fail(NB_ERR_INVALID, "out of host memory");
  t->E = E; t->device = device; t->n_weights = (int)n_weights;
  for (int e = 0; e < E; ++e) { t->G[e][0] = G[2 * e]; t->G[e][1] = G[2 * e + 1]; t->h[e] = h[e]; }
  NB_CUDA(nb::alloc(t->d_weights, (size_t)n_weights));
  NB_CUDA(nb::alloc(t->d_m, (size_t)n_weights));
  NB_CUDA(nb::alloc(t->d_v, (size_t)n_weights));
  NB_CUDA(nb::alloc(t->d_losses, (size_t)4));
  NB_CUDA(cudaMemcpy(t->d_weights.get(), weights, (size_t)n_weights * sizeof(float), cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemset(t->d_m.get(), 0, (size_t)n_weights * sizeof(float)));
  NB_CUDA(cudaMemset(t->d_v.get(), 0, (size_t)n_weights * sizeof(float)));
  *out = t.release();
  return NB_OK;
}

int nb_dune_train_destroy(nb_dune_train_t* t) {
  if (!t) return NB_OK;
  cudaSetDevice(t->device);
  delete t;
  return NB_OK;
}

int nb_dune_train_epoch(nb_dune_train_t* t, const float* pts, const float* mu, const float* dist, int64_t n, int32_t batch, const float* thetas,
                        float lr, int32_t validate, double* losses, void* stream) {
  if (!t || !pts || !mu || !dist || !thetas || !losses) return fail(NB_ERR_INVALID, "nb_dune_train_epoch: null argument");
  if (n < 1 || batch < 1 || batch > nb::kTrainThreads) return fail(NB_ERR_INVALID, "nb_dune_train_epoch: n >= 1 and 1 <= batch_size <= %d required", nb::kTrainThreads);
  NB_CUDA(cudaSetDevice(t->device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t nbatch = (size_t)((n + batch - 1) / batch);
  if (nbatch > t->thetas_cap) {
    t->thetas_cap = 0;
    NB_CUDA(nb::alloc(t->d_thetas, nbatch));
    t->thetas_cap = nbatch;
  }
  NB_CUDA(cudaMemcpyAsync(t->d_thetas.get(), thetas, nbatch * sizeof(float), cudaMemcpyHostToDevice, st));
  nb::DuneTrainParams prm;
  prm.pts = pts; prm.mu = mu; prm.dist = dist; prm.thetas = t->d_thetas.get();
  prm.weights = t->d_weights.get(); prm.adam_m = t->d_m.get(); prm.adam_v = t->d_v.get(); prm.losses = t->d_losses.get();
  prm.n = (int)n; prm.batch = batch; prm.E = t->E; prm.validate = validate ? 1 : 0;
  prm.step0 = t->steps;
  prm.lr = lr; prm.beta1 = 0.9f; prm.beta2 = 0.999f; prm.eps = 1e-8f; prm.weight_decay = 1e-4f;  // Adam(lr, weight_decay=1e-4), dune_train.py:72
  for (int e = 0; e < nb::kMaxEdges; ++e) { prm.G[e][0] = t->G[e][0]; prm.G[e][1] = t->G[e][1]; prm.h[e] = t->h[e]; }
  const size_t smem = nb::dune_train_smem_bytes(t->E);
  NB_CUDA(cudaFuncSetAttribute(nb::dune_train_epoch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  nb::dune_train_epoch_kernel<<<1, nb::kTrainThreads, smem, st>>>(prm);
  ++nb::launches;
  NB_CUDA(cudaGetLastError());
  double sums[4];
  NB_CUDA(cudaMemcpyAsync(sums, t->d_losses.get(), sizeof(sums), cudaMemcpyDeviceToHost, st));
  NB_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < 4; ++i) losses[i] = sums[i] / (double)nbatch;  // mean over the batches, like train_one_epoch (:322-327)
  if (!validate) t->steps += (long long)nbatch;
  return NB_OK;
}

int nb_dune_train_get_weights(nb_dune_train_t* t, float* weights) {
  if (!t || !weights) return fail(NB_ERR_INVALID, "nb_dune_train_get_weights: null argument");
  NB_CUDA(cudaSetDevice(t->device));
  NB_CUDA(cudaMemcpy(weights, t->d_weights.get(), (size_t)t->n_weights * sizeof(float), cudaMemcpyDeviceToHost));
  return NB_OK;
}

// ---- initial path (SURVEY 8f row 1) ---------------------------------------------------------------------------------
int nb_ipath_create(const nb_ipath_config* cfg, nb_ipath_t** out) {
  if (!cfg || !out) return fail(NB_ERR_INVALID, "nb_ipath_create: null argument");
  if (cfg->receding < 1 || cfg->receding > nb::kIpathMaxT) return fail(NB_ERR_INVALID, "receding = %d outside [1, %d]", cfg->receding, nb::kIpathMaxT);
  if (cfg->kinematics < 0 || cfg->kinematics > 2) return fail(NB_ERR_INVALID, "kinematics currently only supports diff, acker or omni");
  if (cfg->kinematics == NB_KIN_ACKER && !(cfg->wheelbase > 0)) return fail(NB_ERR_INVALID, "acker needs a positive wheelbase");
  if (cfg->max_envs < 1 || !(cfg->step_time > 0)) return fail(NB_ERR_INVALID, "max_envs / step_time must be positive");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || cfg->device >= ndev)
    return fail(NB_ERR_NO_DEVICE, "no CUDA device available: neupan_b200 has no CPU fallback");
  NB_CUDA(cudaSetDevice(cfg->device));
  std::unique_ptr<nb_ipath> p(new (std::nothrow) nb_ipath());
  if (!p) return fail(NB_ERR_INVALID, "out of host memory");
  p->cfg = *cfg;
  NB_CUDA(nb::alloc(p->d_env_curve_begin, (size_t)cfg->max_envs + 1));
  NB_CUDA(nb::alloc(p->d_interval, (size_t)cfg->max_envs));
  NB_CUDA(nb::alloc(p->d_curve_index, (size_t)cfg->max_envs));
  NB_CUDA(nb::alloc(p->d_point_index, (size_t)cfg->max_envs));
  NB_CUDA(nb::alloc(p->d_arrive_flag, (size_t)cfg->max_envs));
  *out = p.release();
  return NB_OK;
}

int nb_ipath_destroy(nb_ipath_t* p) {
  if (!p) return NB_OK;
  cudaSetDevice(p->cfg.device);
  delete p;
  return NB_OK;
}

int nb_ipath_reset_async(nb_ipath_t* p, void* stream) {
  if (!p) return fail(NB_ERR_INVALID, "nb_ipath_reset: null handle");
  NB_CUDA(cudaSetDevice(p->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  NB_CUDA(cudaMemsetAsync(p->d_curve_index.get(), 0, sizeof(int32_t) * p->cfg.max_envs, st));
  NB_CUDA(cudaMemsetAsync(p->d_point_index.get(), 0, sizeof(int32_t) * p->cfg.max_envs, st));
  NB_CUDA(cudaMemsetAsync(p->d_arrive_flag.get(), 0, sizeof(int32_t) * p->cfg.max_envs, st));
  return NB_OK;
}

int nb_ipath_reset(nb_ipath_t* p) {
  if (int rc = nb_ipath_reset_async(p, nullptr)) return rc;
  NB_CUDA(cudaStreamSynchronize(nullptr));
  return NB_OK;
}

int nb_ipath_set_paths(nb_ipath_t* p, int32_t B, const double* points, int64_t P, const int32_t* curve_begin, int32_t C,
                       const int32_t* env_curve_begin, const double* interval) {
  if (!p || !points || !curve_begin || !env_curve_begin || !interval) return fail(NB_ERR_INVALID, "nb_ipath_set_paths: null argument");
  if (B < 1 || B > p->cfg.max_envs) return fail(NB_ERR_CAPACITY, "B = %d outside [1, max_envs = %d]", B, p->cfg.max_envs);
  if (P < 1 || C < B) return fail(NB_ERR_INVALID, "every environment needs at least one curve with one point (P = %lld, C = %d)", (long long)P, C);
  if (env_curve_begin[0] != 0 || env_curve_begin[B] != C || curve_begin[0] != 0 || curve_begin[C] != P)
    return fail(NB_ERR_INVALID, "curve_begin / env_curve_begin do not cover the points");
  for (int b = 0; b < B; ++b)
    if (env_curve_begin[b + 1] <= env_curve_begin[b]) return fail(NB_ERR_INVALID, "environment %d has no curve", b);
  for (int c = 0; c < C; ++c)
    if (curve_begin[c + 1] <= curve_begin[c]) return fail(NB_ERR_INVALID, "curve %d is empty", c);
  NB_CUDA(cudaSetDevice(p->cfg.device));
  p->d_pts.reset();
  p->d_curve_begin.reset();
  NB_CUDA(nb::alloc(p->d_pts, (size_t)P * 4));
  NB_CUDA(nb::alloc(p->d_curve_begin, (size_t)C + 1));
  NB_CUDA(cudaMemcpy(p->d_pts.get(), points, sizeof(double) * 4 * P, cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(p->d_curve_begin.get(), curve_begin, sizeof(int32_t) * (C + 1), cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(p->d_env_curve_begin.get(), env_curve_begin, sizeof(int32_t) * (B + 1), cudaMemcpyHostToDevice));
  NB_CUDA(cudaMemcpy(p->d_interval.get(), interval, sizeof(double) * B, cudaMemcpyHostToDevice));
  p->B = B; p->P = P;
  return nb_ipath_reset(p);
}

int nb_ipath_step_ex(nb_ipath_t* p, int32_t B, const int32_t* env_index, const double* states, const float* cur_vel, double ref_speed,
                     float* nom_s, float* nom_u, float* ref_s, float* ref_us, int32_t* arrived, void* stream) {
  if (!p || !states || !cur_vel || !nom_s || !nom_u || !ref_s || !ref_us || !arrived) return fail(NB_ERR_INVALID, "nb_ipath_step: null argument");
  if (!p->d_pts) return fail(NB_ERR_INVALID, "initial path is not set (nb_ipath_set_paths)");
  if (env_index ? B < 1 : B != p->B) {
    if (env_index) return fail(NB_ERR_INVALID, "nb_ipath_step_ex: B = %d rows must be positive", B);
    return fail(NB_ERR_INVALID, "B = %d but the paths were set for %d environments", B, p->B);
  }
  NB_CUDA(cudaSetDevice(p->cfg.device));
  nb::IpathParams prm;
  prm.B = B; prm.T = p->cfg.receding; prm.kinematics = p->cfg.kinematics; prm.loop = p->cfg.loop;
  prm.ind_range = p->cfg.ind_range; prm.arrive_index_threshold = p->cfg.arrive_index_threshold;
  prm.dt = p->cfg.step_time; prm.L = p->cfg.wheelbase; prm.arrive_threshold = p->cfg.arrive_threshold; prm.close_threshold = p->cfg.close_threshold;
  prm.ref_speed = ref_speed;
  prm.pts = p->d_pts.get(); prm.curve_begin = p->d_curve_begin.get(); prm.env_curve_begin = p->d_env_curve_begin.get();
  prm.interval = p->d_interval.get(); prm.curve_index = p->d_curve_index.get(); prm.point_index = p->d_point_index.get();
  prm.arrive_flag = p->d_arrive_flag.get();
  prm.states = states; prm.cur_vel = cur_vel; prm.nom_s = nom_s; prm.nom_u = nom_u; prm.ref_s = ref_s; prm.ref_us = ref_us; prm.arrived = arrived;
  prm.env_index = env_index; prm.n_env = p->B;
  auto* kernel = env_index ? nb::ipath_step_kernel<true> : nb::ipath_step_kernel<false>;
  kernel<<<(B + 63) / 64, 64, 0, (cudaStream_t)stream>>>(prm);
  ++nb::launches;
  NB_CUDA(cudaGetLastError());
  return NB_OK;
}

int nb_ipath_step(nb_ipath_t* p, int32_t B, const double* states, const float* cur_vel, double ref_speed,
                  float* nom_s, float* nom_u, float* ref_s, float* ref_us, int32_t* arrived, void* stream) {
  return nb_ipath_step_ex(p, B, nullptr, states, cur_vel, ref_speed, nom_s, nom_u, ref_s, ref_us, arrived, stream);
}

int nb_ipath_read_state(nb_ipath_t* p, int32_t B, int32_t* curve_index, int32_t* point_index, int32_t* arrive_flag,
                        double* points_host, void* stream) {
  if (!p) return fail(NB_ERR_INVALID, "nb_ipath_read_state: null handle");
  if (B != p->B) return fail(NB_ERR_INVALID, "B = %d but the paths were set for %d environments", B, p->B);
  NB_CUDA(cudaSetDevice(p->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  if (curve_index) NB_CUDA(cudaMemcpyAsync(curve_index, p->d_curve_index.get(), sizeof(int32_t) * B, cudaMemcpyDeviceToDevice, st));
  if (point_index) NB_CUDA(cudaMemcpyAsync(point_index, p->d_point_index.get(), sizeof(int32_t) * B, cudaMemcpyDeviceToDevice, st));
  if (arrive_flag) NB_CUDA(cudaMemcpyAsync(arrive_flag, p->d_arrive_flag.get(), sizeof(int32_t) * B, cudaMemcpyDeviceToDevice, st));
  if (points_host) {
    NB_CUDA(cudaMemcpyAsync(points_host, p->d_pts.get(), sizeof(double) * 4 * p->P, cudaMemcpyDeviceToHost, st));
    NB_CUDA(cudaStreamSynchronize(st));
  }
  return NB_OK;
}

}  // extern "C"
