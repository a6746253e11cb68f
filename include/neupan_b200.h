/*
 * neupan_b200 -- C ABI of the H100-native (sm_90a) PAN hot path (libneupan_b200.so).
 *
 * The reference (hanruihua/NeuPAN) has no FFI: its boundary for this path is the Python class
 * neupan.blocks.PAN (neupan/blocks/pan.py:27-147), constructed at neupan/neupan.py:84 and called
 * at neupan/neupan.py:129-131.  Each entry point below names the reference interface it replaces.
 * Plain pointers and sizes only -- no torch / C++ types.  All tensors are float32, row-major,
 * batch-leading ("B" = number of independent environments; the reference is the B == 1 case
 * without the leading axis).  Unless a function says "host", every data pointer is a DEVICE
 * pointer on the handle's device, and work is enqueued on `stream` (a cudaStream_t passed as
 * void*; NULL = the legacy default stream) without synchronising.
 *
 * Return value: 0 on success, a negative NB_ERR_* code otherwise; nb_last_error() gives the text
 * (thread-local).  A per-environment solver problem never fails the call: it is reported in the
 * `status` output instead (the reference lets solver exceptions propagate, nrmp.py:144).
 */
#ifndef NEUPAN_B200_H
#define NEUPAN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NB_VERSION 1

enum { NB_KIN_DIFF = 0, NB_KIN_ACKER = 1, NB_KIN_OMNI = 2 };

enum {
  NB_OK = 0,
  NB_ERR_INVALID = -1,   /* bad argument (ValueError / AssertionError in the reference) */
  NB_ERR_CUDA = -2,      /* CUDA runtime error */
  NB_ERR_CAPACITY = -3,  /* B or N above what the handle was created for */
  NB_ERR_NO_DEVICE = -4  /* no usable CUDA device: there is NO CPU fallback */
};

/* per-environment status bits written by the NRMP solve */
enum {
  NB_STATUS_OK = 0,
  NB_STATUS_MAXITER = 1,     /* interior point method hit its iteration cap */
  NB_STATUS_NUMERIC = 2,     /* non-finite value / failed factorisation */
  NB_STATUS_INFEASIBLE = 4   /* empty bounds (d_min > d_max, max_speed <= 0, max_acce <= 0); d_min == d_max is feasible: D is fixed */
};

typedef struct nb_pan nb_pan_t; /* opaque; owns weights, workspaces and the per-env state of
                                   PAN.current_nom_values (pan.py:100-105) */

/* Everything PAN.__init__ (pan.py:43-107), NRMP.__init__ (nrmp.py:35-112) and robot.__init__
 * (neupan/robot/robot.py:32-71) fix at construction time. */
typedef struct {
  int32_t receding;       /* T            pan.py:45                                  */
  int32_t kinematics;     /* NB_KIN_*     robot.py:34,60                             */
  int32_t edge_dim;       /* E = rows of G (3..8)   dune.py:47                       */
  int32_t iter_num;       /* K            pan.py:48                                  */
  int32_t nrmp_max_num;   /* M (0 => no_obs, pan.py:85); receding <= 32, M <= 32 and receding * M <= 256 */
  int32_t max_envs;       /* capacity: largest B of any later call                   */
  int32_t max_points;     /* capacity: largest N of any later call (after decimation).  The exact and warpgroup screening DUNE
                             kernels hold the operand image, two 16 KB tiles and per-point keys / mu in shared memory: on an H100
                             (227 KB per block) N up to 6981 at E = 4, 4188 at E = 8 (M = 10); a larger N fails at launch with
                             NB_ERR_CAPACITY ("N=... needs ... B of shared memory"). */
  int32_t device;         /* CUDA device ordinal                                     */
  float iter_threshold;   /* pan.py:52; <= 0 never stops early                       */
  /* Python floats in the reference (float64 constants of the convex program): */
  double step_time;       /* dt           pan.py:46                                  */
  double wheelbase;       /* L (acker)    robot.py:58                                */
  double max_speed[2];    /* robot.py:61 (INFINITY allowed; acker steering is clipped to 1.57 by the caller, robot.py:63-66) */
  double max_acce[2];     /* robot.py:62 (per second; multiplied by dt inside, robot.py:69) */
  double ro_obs, bk;      /* nrmp.py:100-101                                         */
  /* float32 tensors in the reference (cvxpy Parameters): */
  float q_s[3];           /* nrmp.py:83-95 (scalar q_s => three equal entries)       */
  float p_u, eta, d_max, d_min; /* nrmp.py:79-98                                     */
} nb_pan_config;

/* Number of float32 values of an ObsPointNet checkpoint with E outputs
 * (obs_point_net.py:31-46): 4512 + 33*E  (4644 for E = 4). */
int64_t nb_weight_count(int32_t edge_dim);

/* Replaces PAN.__init__ -> NRMP.__init__ + DUNE.__init__/load_model (pan.py:43-107,
 * dune.py:31-54,131-144).  `weights` (HOST) holds the state_dict tensors concatenated in key
 * order MLP.{0,1,3,5,6,8,10,11,13}.{weight,bias}; G (E x 2) and h (E) are HOST arrays from
 * gen_inequal_from_vertex (util/__init__.py:161-206). */
int nb_pan_create(const nb_pan_config* cfg, const float* weights, int64_t n_weights,
                  const float* G, const float* h, nb_pan_t** out);
int nb_pan_destroy(nb_pan_t* pan);

/* Replaces PAN.forward (pan.py:109-147): up to K iterations of {point flow -> DUNE -> NRMP ->
 * stop criterion} for B environments.
 *   nom_s (B,3,T+1)  nom_u (B,2,T)  ref_s (B,3,T+1)  ref_us (B,T)
 *   points (B,2,N) or NULL (no obstacle points: pan.py:130-138 else-branch)
 *   velocities (B,2,N) or NULL (static points, pan.py:168-169)
 *   num_points (B) int32 or NULL: valid point count per env (ragged batches; <= N)
 * outputs: out_s (B,3,T+1)  out_u (B,2,T)  out_d (B,T) [nom_distance, zeros in no_obs mode]
 *   out_min_distance (B) [DUNE.min_distance, dune.py:97-98; +inf without points]
 *   out_iters (B) int32 or NULL: iterations executed per env;  out_status (B) int32 or NULL.
 * Inputs are never modified; outputs may not alias inputs. */
int nb_pan_forward(nb_pan_t* pan, int32_t B, int32_t N,
                   const float* nom_s, const float* nom_u, const float* ref_s, const float* ref_us,
                   const float* points, const float* velocities, const int32_t* num_points,
                   float* out_s, float* out_u, float* out_d, float* out_min_distance,
                   int32_t* out_iters, int32_t* out_status, void* stream);

/* Same call with HOST buffers (what neupan.forward does around PAN: np_to_tensor / tensor_to_np,
 * neupan/neupan.py:123-135): stages through the handle's device workspace on `stream` and
 * returns after the results have landed in the host buffers. */
int nb_pan_forward_host(nb_pan_t* pan, int32_t B, int32_t N,
                        const float* nom_s, const float* nom_u, const float* ref_s, const float* ref_us,
                        const float* points, const float* velocities, const int32_t* num_points,
                        float* out_s, float* out_u, float* out_d, float* out_min_distance,
                        int32_t* out_iters, int32_t* out_status, void* stream);

/* HOST inputs (pinned memory for a real overlap), DEVICE outputs, asynchronous on `stream` like nb_pan_forward: the inputs are uploaded
 * on an internal copy stream in environment chunks and the first DUNE pass of a chunk starts as soon as its points have landed, so
 * the upload of the cloud hides behind the first PAN iteration (the callers that keep results on the device -- e.g. to exchange them
 * between GPUs before they travel back -- use this one; nb_pan_forward_host is this call plus the download and a synchronise). */
int nb_pan_forward_h2d(nb_pan_t* pan, int32_t B, int32_t N,
                        const float* nom_s, const float* nom_u, const float* ref_s, const float* ref_us,
                        const float* points, const float* velocities, const int32_t* num_points,
                        float* out_s, float* out_u, float* out_d, float* out_min_distance,
                        int32_t* out_iters, int32_t* out_status, void* stream);

/* Replaces NRMP.update_adjust_parameters_value (nrmp.py:171-217). */
int nb_pan_set_adjust(nb_pan_t* pan, const float q_s[3], float p_u, float eta, float d_max, float d_min);
/* iter_num / iter_threshold are plain attributes in the reference (pan.py:63-64). */
int nb_pan_set_iteration(nb_pan_t* pan, int32_t iter_num, float iter_threshold);

/* Implementation switches (no reference counterpart).  NB_OPT_DUNE_KERNEL: 2 (the handle's initial value; the Python mirror selects 4) =
 * warpgroup DUNE kernel on every point (wgmma with a shared-memory operand / output tile, fp16 hi/lo split, fp32 accumulate);
 * 4 = wgmma with screening: a single-pass fp16 interval pass over all points, the exact network only for the <= 32 points
 * per (environment, step) that can be among the M closest, the exact kernel for the items the screen cannot narrow down -- the same
 * selection and values as 2, bit for bit (csrc/dune_screen_kernel.cuh).  Other values are refused with NB_ERR_INVALID.
 * NB_OPT_OVERLAP: 1..4 = number of environment sub-batches pipelined on internal streams so that the DUNE kernels
 * of one sub-batch share the SMs with the NRMP kernel of another (results are identical; envs are independent; batches with
 * fewer than 64 environments per part are not split).  The handle starts with 2: the straggler tail of one half's NRMP launch
 * and the small kernels between the big ones run under the other half's DUNE pass.
 * NB_OPT_NRMP_WARM: 1 = inside one nb_pan_forward the NRMP solve of PAN iteration k > 0 starts from the solution of
 * iteration k-1 of the same environment (fewer interior point iterations on average, same optimum to the solver tolerance;
 * a warm start that is not converging by its 12th iteration is abandoned for a cold one); 0 (default) = every solve starts
 * cold.  The first solve of every call is always cold, so results never depend on earlier calls.
 * NB_OPT_DIFFERENTIABLE: 1 = every NRMP solve of nb_pan_forward also stores what nb_pan_backward needs (one extra factorisation
 * at the optimum + ~5 KB per environment and iteration); 0 (default) = inference only.
 * NB_OPT_DUNE_SCREEN_MMA (with NB_OPT_DUNE_KERNEL = 4): 1 (default) = the screening pass runs on warp-level mma.sync with the
 * activations in registers (csrc/dune_screen_mma_kernel.cuh; clouds of at most 1024 points, larger ones take the wgmma pass), 0 = on
 * wgmma (csrc/dune_screen_kernel.cuh).  Same candidate contract, same final results (the refine / exact kernels are wgmma either way).
 * NB_OPT_DUNE_SKIP_T0 (with NB_OPT_DUNE_KERNEL = 4): 1 (default) = PAN iterations k > 0 of one nb_pan_forward do not re-evaluate the
 * step-0 items: nom_s[:, 0] is the fixed initial state (robot.py:234), so their inputs and results are those of iteration 0, which
 * stand in the selection buffers; 0 = evaluate them in every iteration (identical results).
 * NB_OPT_DUNE_SCREEN_TABLE (with NB_OPT_DUNE_KERNEL = 4 and the mma.sync screen): 1 (default) = the screen looks each point's distance
 * and error radius up in a table of the network's distance over the robot frame, built once per handle when both are first selected
 * (csrc/dune_table_kernel.cuh; points outside the table take the network; a table less than twice as accurate as the handle's
 * bound c_mu is not kept, and the network screens every point); 0 = every point runs the single-pass fp16 network.  Same final
 * results, bit for bit. */
enum { NB_OPT_DUNE_KERNEL = 1, NB_OPT_OVERLAP = 2, NB_OPT_NRMP_WARM = 3, NB_OPT_DIFFERENTIABLE = 4, NB_OPT_DUNE_SCREEN_MMA = 5, NB_OPT_DUNE_SKIP_T0 = 6,
       NB_OPT_DUNE_SCREEN_TABLE = 7 };
int nb_pan_set_option(nb_pan_t* pan, int32_t option, int32_t value);

/* Replaces the backward pass of the reference's differentiable solve (CvxpyLayer, nrmp.py:144; used by LON,
 * example/LON/LON_corridor.py:94 `loss.backward()`): given dL/d(out_s) (B,3,T+1), dL/d(out_u) (B,2,T), dL/d(out_d) (B,T) of the
 * LAST nb_pan_forward (made with NB_OPT_DIFFERENTIABLE = 1; any gradient pointer may be NULL = zeros) it writes
 * grad_theta (B,7) = dL/d(q_s[0], q_s[1], q_s[2], p_u, eta, d_max, d_min) per environment (a scalar q_s is the sum of the
 * first three; parameters shared by the batch are the sum over environments).  Like the reference, the gradient flows through
 * every PAN iteration's solve: directly through the adjust parameters (incl. gamma_a = q_s ref_s, gamma_b = p_u ref_us,
 * nrmp.py:156-159) and from iteration k to k-1 through `nom_s` (the proximal term and nothing else: A, B, C, fa, fb are rebuilt
 * from detached values in the reference, robot.py:272-316, dune.py:78-95).  ref_s / ref_us are the tensors of the forward call. */
int nb_pan_backward(nb_pan_t* pan, int32_t B, const float* ref_s, const float* ref_us,
                    const float* grad_s, const float* grad_u, const float* grad_d, float* grad_theta, void* stream);

/* Forget PAN.current_nom_values (pan.py:100-105) of all environments.  (The reference's
 * neupan.reset() does NOT do this, neupan/neupan.py:288-294; exposed for tests and for
 * re-using a handle on a new batch.) */
int nb_pan_reset_state(nb_pan_t* pan);                      /* legacy default stream, returns after completion */
int nb_pan_reset_state_async(nb_pan_t* pan, void* stream);   /* ordered with the forwards enqueued on `stream` */
/* The same for the environments b < B whose mask[b] (DEVICE int32, B <= max_envs) is non-zero; the others keep their state.  One
 * small kernel on `stream`, no synchronisation (what a batched closed loop calls when some environments start a new episode).  With
 * every mask entry 1 and B = max_envs it clears exactly what nb_pan_reset_state_async clears. */
int nb_pan_reset_envs_async(nb_pan_t* pan, int32_t B, const int32_t* mask, void* stream);

/* The sorted selections of the last executed iteration, what DUNE.forward returns restricted to
 * the first M columns (dune.py:100-104): mu (B,T+1,M,E) lam (B,T+1,M,2) points (B,T+1,M,2)
 * distance (B,T+1,M) count (B) int32 [= min(num_points, M)].  Any pointer may be NULL.
 * sel_points[:,0] is NRMP.points / PAN.nrmp_points (nrmp.py:135-138, pan.py:262-268). */
int nb_pan_read_selection(nb_pan_t* pan, int32_t B, float* sel_mu, float* sel_lam, float* sel_points,
                          float* sel_distance, int32_t* sel_count, void* stream);

/* Screening statistics accumulated since the last reset (HOST outputs; synchronises the device): max_error_ratio[0] = the largest
 * |screened - exact distance| / sum_e |G_e p0 - h_e| over all refined candidates, [1] = the handle's bound c_mu it must stay below
 * (4 x the error measured at calibration, when NB_OPT_DUNE_KERNEL = 4 is first selected), [2] = that calibration measurement;
 * counts[0] = items sent to the exact kernel, counts[1] = candidates refined, counts[2] = items screened. */
int nb_pan_read_screen_stats(nb_pan_t* pan, float* max_error_ratio, int32_t* counts, int32_t reset);
/* The two-level table path of the one-warp-per-item screen since the last reset: counts[0] = points that survived the coarse bound
 * table (summed over the items that took the path), counts[1] = items that tried the path and took the one-level path instead (a
 * point outside the table, or more survivors than the path holds); both stay 0 with NB_SCREEN_COARSE=0.  Reset separately from
 * nb_pan_read_screen_stats. */
int nb_pan_read_screen_coarse(nb_pan_t* pan, int32_t counts[2], int32_t reset);
/* The screen's distance table (all zero while none is built): info[0] = cell side h (m), [1] = half-width of the covered square (m),
 * [2] = device bytes (0: built, but not kept: [4] > c_mu / 2), [3] = build time (ms, host clock around the synchronised build), [4] = the largest |table - network| /
 * sum_e |G_e p - h_e| on the 4 x 4 sub-grid of every cell. */
int nb_pan_read_screen_table(nb_pan_t* pan, float info[5]);

/* Diagnostics of the last executed NRMP solve (nb_pan_forward or nb_nrmp_forward): interior point iterations per env (B) int32. */
int nb_pan_read_diagnostics(nb_pan_t* pan, int32_t B, int32_t* ipm_iterations, void* stream);

/* ---- the two halves, exposed separately (parity tests, profiling) ------------------------ */

/* PAN.generate_point_flow + DUNE.forward (pan.py:150-212, dune.py:58-127) for B envs, keeping the
 * M closest points per (env, step) in ascending distance order.  Results land in the handle
 * (read them with nb_pan_read_selection); out_min_distance (B) may be NULL. */
int nb_dune_forward(nb_pan_t* pan, int32_t B, int32_t N, const float* nom_s, const float* points,
                    const float* velocities, const int32_t* num_points, float* out_min_distance, void* stream);

/* NRMP.forward (nrmp.py:114-150) for B envs on explicit obstacle coefficients:
 * fa (B,T,M,2) = lam^T rows, fb (B,T,M) = lam^T p + mu^T h (nrmp.py:220-261); NULL => zeros. */
int nb_nrmp_forward(nb_pan_t* pan, int32_t B, const float* nom_s, const float* nom_u, const float* ref_s,
                    const float* ref_us, const float* fa, const float* fb,
                    float* out_s, float* out_u, float* out_d, int32_t* out_status, void* stream);

/* ---- lidar scan -> obstacle points (the producer of `points`; SURVEY 8f "next" row 2) -------------------------- */

/* The `scan` dict and the arguments of neupan.scan_to_point / scan_to_point_velocity (neupan/neupan.py:173-281). */
typedef struct nb_scan_config {
  double angle_min, angle_max;   /* scan["angle_min"], scan["angle_max"]: beam i sits at linspace(min, max, R)[i]      */
  double range_min, range_max;   /* kept: range < range_max - 0.02 and range > (mode 1: >=) range_min                  */
  double scan_offset[3];         /* sensor pose in the robot frame                                                     */
  double angle_range[2];         /* kept: angle_range[0] < angle < angle_range[1]                                      */
  int32_t down_sample;           /* the [:, ::down_sample] stride over the kept points (>= 1)                          */
  int32_t velocity_mode;         /* 0: scan_to_point (offset applied as s_R p + s_t, neupan.py:216-217);
                                    1: scan_to_point_velocity (s_R^T (p - s_t), range >= range_min, neupan.py:258-273) */
} nb_scan_config;

/* B scans of R beams each -> points (B,2,max_points) float32 in the world frame, their per-beam velocities (optional)
 * and the number of valid columns per environment; more than max_points survivors are decimated exactly like
 * PAN.generate_point_flow does (pan.py:171-174 -> downsample_decimation: columns linspace(0, n-1, max_points).astype(int)).
 * All pointers are DEVICE pointers; ranges (B,R) float32, velocity (B,2,R) float32 or NULL, states (B,3) float64
 * [x, y, theta].  The outputs are exactly what nb_pan_forward takes as (points, velocities, num_points) with N = max_points.
 * A scan with no surviving beam yields count 0 (the reference returns None). */
int nb_scan_to_points(int32_t B, int32_t R, const float* ranges, const float* velocity, const double* states,
                      const nb_scan_config* cfg, int32_t max_points, float* points, float* velocities_out,
                      int32_t* counts, void* stream);

/* ---- initial path: check_arrive + generate_nom_ref_state for B environments (SURVEY 8f "next" row 1) -------------- */

/* The numbers of InitialPath.__init__ (neupan/blocks/initial_path.py:35-64) the per-step work needs. */
typedef struct nb_ipath_config {
  int32_t receding;                /* T */
  int32_t kinematics;              /* NB_KIN_*: selects the motion_predict_model (initial_path.py:386-444) */
  int32_t loop;                    /* restart at the first curve when the last one is finished (:262-269) */
  int32_t ind_range;               /* window of closest_point (:166-183), reference default 10 */
  int32_t arrive_index_threshold;  /* check_curve_arrive (:282-290), reference default 1 */
  int32_t max_envs;
  int32_t device;
  int32_t reserved_;
  double step_time;
  double wheelbase;                /* robot.L, acker only */
  double arrive_threshold;         /* reference default 0.1 */
  double close_threshold;          /* reference default 0.1 */
} nb_ipath_config;

typedef struct nb_ipath nb_ipath_t;

int nb_ipath_create(const nb_ipath_config* cfg, nb_ipath_t** out);
int nb_ipath_destroy(nb_ipath_t* ip);

/* InitialPath.set_initial_path (initial_path.py:128-144) for B environments, already split by gear
 * (split_path_with_gear, :294-317): HOST arrays; points (P,4) float64 rows [x, y, theta, gear], all curves of all
 * environments back to back; curve_begin (C+1) offsets into points; env_curve_begin (B+1) offsets into curve_begin;
 * interval (B) = cal_average_interval of each environment's whole path (:146-164; computed by the caller, whose
 * math.hypot it must reproduce).  Resets curve_index / point_index / arrive_flag.  The handle keeps a MUTABLE device copy
 * of the points: like the reference it rewrites path headings while generating references (:99,112,191-192). */
int nb_ipath_set_paths(nb_ipath_t* ip, int32_t B, const double* points, int64_t P, const int32_t* curve_begin, int32_t C,
                       const int32_t* env_curve_begin, const double* interval);

/* One control step for B environments (neupan.forward before PAN, neupan/neupan.py:114-121):
 *   arrived[b] = InitialPath.check_arrive(state_b)                              (initial_path.py:251-292)
 *   nom_s, nom_u, ref_s, ref_us = InitialPath.generate_nom_ref_state(state_b, cur_vel_b, ref_speed)   (:68-126)
 * DEVICE pointers: states (B,3) float64; cur_vel (B,2,T) float32 (the velocities PAN returned at the previous step);
 * outputs float32 in nb_pan_forward's layouts: nom_s (B,3,T+1), nom_u (B,2,T), ref_s (B,3,T+1), ref_us (B,T);
 * arrived (B) int32.  Environments that have arrived get zero trajectories (the reference returns before generating). */
int nb_ipath_step(nb_ipath_t* ip, int32_t B, const double* states, const float* cur_vel, double ref_speed,
                  float* nom_s, float* nom_u, float* ref_s, float* ref_us, int32_t* arrived, void* stream);
/* The same with env_index (B) int32 DEVICE: row b (states, cur_vel and every output) steps the path and the persistent indices of
 * environment env_index[b] of a handle that holds paths for S environments (nb_ipath_set_paths with S); B is any positive count,
 * and rows must name distinct environments.  An index outside 0..S-1 gives its row arrived = 1 and zero trajectories.  NULL is
 * the identity: exactly nb_ipath_step (B must equal S). */
int nb_ipath_step_ex(nb_ipath_t* ip, int32_t B, const int32_t* env_index, const double* states, const float* cur_vel, double ref_speed,
                     float* nom_s, float* nom_u, float* ref_s, float* ref_us, int32_t* arrived, void* stream);

/* neupan.reset (neupan/neupan.py:287-294): point_index = curve_index = 0, arrive_flag = False for every environment.
 * The path headings rewritten so far stay as they are (as in the reference). */
int nb_ipath_reset(nb_ipath_t* ip);                       /* legacy default stream, returns after completion */
int nb_ipath_reset_async(nb_ipath_t* ip, void* stream);   /* ordered with the steps enqueued on `stream` */

/* Persistent per-environment indices and a copy of the (mutated) path points; any pointer may be NULL.  DEVICE pointers
 * for the indices (B) int32, HOST pointer for points (P,4) float64 (synchronises `stream`). */
int nb_ipath_read_state(nb_ipath_t* ip, int32_t B, int32_t* curve_index, int32_t* point_index, int32_t* arrive_flag,
                        double* points_host, void* stream);

/* ---- batched 2-D world: lidar scans, moving obstacles and collisions for closed-loop runs ------------------------------ */

/* What the reference's simulator (IR-SIM, example/run_exp.py:27-56, configured by example/<scenario>/<kin>/env.yaml) provides around
 * the planner, for B environments on the device.  The robot is a convex polygon (the planner's robot.vertices, neupan_b200/robot.py);
 * the lidar is the `lidar2d` sensor without noise. */
typedef struct nb_world_config {
  int32_t kinematics;              /* NB_KIN_*: diff (v, omega), acker (v, steering phi), omni (vx, vy)                           */
  int32_t num_beams;               /* R >= 1                                                                                    */
  int32_t max_envs;
  int32_t device;
  int32_t robot_num_vertices;      /* 3..8 */
  int32_t reserved_;
  double step_time;                /* dt of one nb_world_step */
  double wheelbase;                /* robot.L, acker only */
  double angle_min, angle_max;     /* beam i sits at linspace(angle_min, angle_max, R)[i] in the sensor frame                   */
  double range_max;                /* a beam with no crossing closer than range_max reports range_max                          */
  double scan_offset[3];           /* sensor pose in the robot frame                                                            */
  double robot_vertices[16];       /* x0, y0, x1, y1, ...: the convex robot polygon in its own frame                            */
} nb_world_config;

typedef struct nb_world nb_world_t;  /* opaque; owns the scenes, robot states and flags of B environments */

int nb_world_create(const nb_world_config* cfg, nb_world_t** out);
int nb_world_destroy(nb_world_t* w);

/* The scene of every environment (the obstacle, robot and goal sections of env.yaml), HOST arrays, ragged like nb_ipath_set_paths:
 *   obs_begin (B+1) int32   offsets into the obstacle rows; at most 256 obstacles and 2048 polygon edges per environment
 *   obstacles (O,5) float64 rows [cx, cy, vx, vy, radius]: centre, constant world-frame velocity, circle radius (> 0; unused for
 *                           polygons).  An obstacle whose velocity component is non-zero must start inside its rectangle, and
 *                           |v| * step_time must be smaller than the rectangle's extent on that axis.
 *   vert_begin (O+1) int32  offsets into vertices; an empty range is a circle, otherwise a convex polygon of 3..8 vertices
 *   vertices (V,2) float64  polygon vertices relative to the obstacle's centre (motion moves the centre only)
 *   envs (B,10) float64     rows [xmin, ymin, xmax, ymax, start_x, start_y, start_theta, goal_x, goal_y, goal_threshold]: the
 *                           rectangle in which moving obstacles bounce, the robot's initial state and its goal
 * nb_world_check_scenes performs every check of nb_world_set_scenes on the host (NB_ERR_INVALID) without a handle or a device.
 * nb_world_set_scenes (IR-SIM's make_env / env.reset) uploads the scenes, places the robots at their starts and clears the
 * collided / arrived flags; it synchronises the device. */
int nb_world_check_scenes(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obstacles,
                          const int32_t* vert_begin, const double* vertices, const double* envs);
int nb_world_set_scenes(nb_world_t* w, int32_t B, const int32_t* obs_begin, const double* obstacles, const int32_t* vert_begin,
                        const double* vertices, const double* envs);

/* The same with obstacles of any shape: obs_kind (O) int32 HOST, or NULL (every kind 0: exactly nb_world_check_scenes /
 * nb_world_set_scenes, whose checks, messages and uploaded bytes these are).
 *   kind 0   a circle (empty vertex range) or a convex polygon of 3..8 vertices, as above
 *   kind 1   an outline: any simple polygon of 3..16 vertices, convex or not, in either orientation (no zero-length edge, non-zero
 *            area, no two edges that do not share a vertex intersect or touch; O(n^2) per outline).  Its edges are scanned like a
 *            convex polygon's; its clearance is 0 when an outline edge meets a robot edge or either polygon contains the other's
 *            vertex 0 (even-odd / sign tests), else the smallest vertex-edge distance both ways.
 * At most 2048 polygon edges per environment, convex polygons and outlines together. */
int nb_world_check_scenes_ex(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obstacles,
                             const int32_t* vert_begin, const double* vertices, const double* envs, const int32_t* obs_kind);
int nb_world_set_scenes_ex(nb_world_t* w, int32_t B, const int32_t* obs_begin, const double* obstacles, const int32_t* vert_begin,
                           const double* vertices, const double* envs, const int32_t* obs_kind);

/* env.get_lidar_scan() for every environment (the dict's `ranges` and per-beam `velocity`), DEVICE outputs:
 *   ranges (B,R) float32: the first crossing t > 0 of beam i with an obstacle boundary (circle: the quadratic; polygon: every edge);
 *     range_max when there is none closer; the robot's own body is not seen; a sensor inside an obstacle sees the exit crossing
 *   velocity (B,2,R) float32 or NULL: world-frame velocity of the obstacle a beam hit, zero on a miss (neupan.py:252 consumes it)
 *   hit (B,R) int32 or NULL: index of that obstacle within its environment, -1 on a miss; equal t: the lower index
 * FP64 arithmetic, float32 at the store; ranges and velocity are exactly what nb_scan_to_points takes. */
int nb_world_scan(nb_world_t* w, int32_t B, float* ranges, float* velocity, int32_t* hit, void* stream);

/* env.step(action) + env.done() for every environment: obstacles move by v * dt (a moving centre that leaves its rectangle is mirrored
 * back and that velocity component reversed); a robot that has not collided integrates action (B,2) float32 DEVICE with the motion
 * models of initial_path.py:401-444 (diff: (v cos th, v sin th, omega); acker: (v cos th, v sin th, v tan phi / L); omni: (vx, vy), the
 * velocities PlannerBatch returns), FP64 state.  Then the exact Euclidean clearance between the robot polygon and every obstacle
 * (0 when they overlap) and the sticky flags: collided = clearance <= 0 (the robot stops for good: collision_mode 'stop'),
 * arrived = distance to the goal < goal_threshold.  DEVICE outputs, any may be NULL: collided, arrived (B) int32, clearance (B)
 * float32 (min over the obstacles; +inf without obstacles). */
int nb_world_step(nb_world_t* w, int32_t B, const float* action, int32_t* collided, int32_t* arrived, float* clearance, void* stream);

/* env.get_robot_state() and the obstacle states, DEVICE outputs, any may be NULL: states (B,3) float64 [x, y, theta],
 * obstacles (O,5) float64 (the rows of nb_world_set_scenes with the current centres and velocities), collided, arrived (B) int32.
 * Enqueued on `stream` without synchronising. */
int nb_world_read_state(nb_world_t* w, int32_t B, double* states, double* obstacles, int32_t* collided, int32_t* arrived, void* stream);

/* Obstacle behaviours: behaviors (O,13) float64 HOST rows
 *   [kind (0 constant velocity, 1 rvo), vxmax, vymax, acce, factor, speed, wander (0 | 1), goal_x, goal_y (NaN, NaN: draw 0),
 *    goal_threshold, neighbor_range, grid, min_speed]
 * A kind-0 row keeps the obstacle's constant velocity (its other columns are not read).  A kind-1 obstacle is reactive: before every
 * nb_world_step moves anything, it heads for its goal at `speed` and steers around the other obstacles and the robot with a
 * reciprocal velocity obstacle, choosing from a grid of candidate velocities (this project's reading of IR-SIM's `rvo` behaviour,
 * stated in full in csrc/world_rvo_kernel.cuh); with `wander` it draws a new goal in its rectangle on arrival, without it it parks.
 * Goals are drawn from SplitMix64 streams keyed by (seed, environment, obstacle index within it, draw number).
 * Checks (NB_ERR_INVALID, with the obstacle index): kind 0 or 1; finite values (a NaN goal requests draw 0); positive vxmax, vymax,
 * acce, factor, speed, goal_threshold, neighbor_range, grid and min_speed >= 0; at most 64 candidates per axis
 * (ceil(2 min(acce, vmax) / grid)); a reactive obstacle's centre inside its rectangle, vmax * step_time below the rectangle's extent,
 * and an explicit goal inside the rectangle.
 * nb_world_check_behaviors checks scenes and behaviours on the host without a handle or a device.  nb_world_set_behaviors applies
 * them to the current state of a handle's scenes (their current centres) and synchronises the device; nb_world_set_scenes(_ex) makes
 * every obstacle kind 0 again.  A world without a kind-1 obstacle launches nothing more per step than one without behaviours. */
int nb_world_check_behaviors(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obstacles,
                             const int32_t* vert_begin, const double* vertices, const double* envs, const int32_t* obs_kind,
                             const double* behaviors, uint64_t seed);
int nb_world_set_behaviors(nb_world_t* w, int32_t B, const double* behaviors, uint64_t seed);

/* The current goals (O,2) float64 and goal draw counters (O) int32 (the draws made so far), DEVICE outputs, either may be NULL;
 * enqueued on `stream` without synchronising.  NB_ERR_INVALID before nb_world_set_behaviors. */
int nb_world_read_behaviors(nb_world_t* w, int32_t B, double* goals, int32_t* draws, void* stream);

/* Several robots per environment (IR-SIM's robot: section as a list; this project's reading, stated in csrc/world_kernel.cuh):
 *   robots (B*K,6) float64 HOST rows [start x, y, theta, goal x, y, goal_threshold], robot k of environment b at row n = b*K + k.
 * Every robot has the handle's polygon, kinematics and lidar (nb_world_set_fleet_ex below: robots of several types); 1 <= K <= 16.  nb_world_set_fleet (after nb_world_set_scenes(_ex))
 * places the B*K robots at their starts and clears their flags; the env rows' start and goal are then unused; behaviours stay set.
 * nb_world_set_scenes(_ex) returns the handle to one robot per environment.  With a fleet, nb_world_scan, nb_world_step and
 * nb_world_read_state take N = B*K as their count and their per-robot arrays have N rows (ranges (N,R), velocity (N,2,R), hit (N,R),
 * action (N,2), collided / arrived / clearance (N), states (N,3)); obstacle rows and nb_world_read_behaviors are unchanged.
 *   scan    a beam also tests the bodies of the environment's other K-1 robots (the polygon at their current state), never its own;
 *           robot j is hit index O_b + j (O_b: the environment's obstacle count), so at equal t an obstacle wins; its velocity is the
 *           world-frame velocity of the action it integrated in the last step (diff / acker v (cos th, sin th) with the heading before
 *           that step, omni (vx, vy)): 0 before the first step and once it has collided; translation only (omega x r is left out).
 *   step    Jacobi: every robot that has not collided integrates its own action from the state at the start of the step, obstacles
 *           move once per environment; a robot's clearance is the minimum over the obstacles and the other robots (convex-convex,
 *           symmetric bit for bit, so two robots that touch collide in the same step).  collided (sticky) freezes a robot, which
 *           stays in the scene with velocity 0; arrived is per robot and sticky.
 *   rvo     reactive obstacles take every robot of their environment as a neighbour (rows after the obstacles, in robot order).
 * Checks (NB_ERR_INVALID, naming the environment / robot): K in 1..16, finite rows, goal_threshold >= 0, no two start bodies of an
 * environment that overlap or touch (SAT on the host).  nb_world_check_fleet performs them without a handle or a device.
 * nb_world_set_fleet allocates the per-robot arrays once and synchronises the device; scan and step neither allocate nor synchronise.
 * A fleet of K = 1 whose rows repeat the env rows gives exactly the world without a fleet. */
int nb_world_check_fleet(const nb_world_config* cfg, int32_t B, int32_t K, const double* robots);
int nb_world_set_fleet(nb_world_t* w, int32_t B, int32_t K, const double* robots);

/* Mixed fleets: robots of different shapes and kinematics in one world.  A robot type is a body and a motion model; type 0 is the
 * robot of nb_world_config, types 1..T are types[0 .. T) (HOST), at most 4 types per handle (T <= 3).  robot_type (B*K) int32 HOST
 * gives each robot's type (NULL: every robot is type 0).  The lidar (R, angles, range_max, scan_offset) is shared by every type, so
 * every scan has the shape (N,R).  Each robot integrates with its type's kinematics and wheelbase, its body is its type's polygon
 * (what the other robots' beams see, and what its clearances are taken from; robot-robot clearances stay symmetric bit for bit
 * across types), and a reactive obstacle sees it as a circle of its type's circumradius moving with its type's velocity model.  K = 1
 * is allowed: one robot per environment, of any type.
 * Checks (NB_ERR_INVALID) besides those of nb_world_check_fleet: T in 0..3 and types not NULL when T > 0; per type (named): the
 * config polygon's checks (3..8 vertices, finite, convex), a known kinematics, a positive wheelbase for acker; every robot_type in
 * 0..T (naming the environment and robot); the start bodies' overlap test takes each robot's own polygon.
 * nb_world_set_fleet / nb_world_check_fleet are these calls with T = 0 and robot_type = NULL (the same checks, messages and uploaded
 * bytes); nb_world_set_scenes(_ex) returns the handle to one type-0 robot per environment. */
typedef struct nb_world_robot_type {
  int32_t kinematics;              /* NB_KIN_* */
  int32_t num_vertices;            /* 3..8 */
  double wheelbase;                /* acker only */
  double vertices[16];             /* x0, y0, x1, y1, ...: the convex polygon in the robot's frame */
} nb_world_robot_type;

int nb_world_check_fleet_ex(const nb_world_config* cfg, int32_t T, const nb_world_robot_type* types, int32_t B, int32_t K, const double* robots,
                            const int32_t* robot_type);
int nb_world_set_fleet_ex(nb_world_t* w, int32_t T, const nb_world_robot_type* types, int32_t B, int32_t K, const double* robots,
                          const int32_t* robot_type);

/* Occupancy maps (this project's reading of IR-SIM's `world: obstacle_map:`; semantics in csrc/world_kernel.cuh): a static grid of
 * width x height square cells of side `resolution` (m), origin (x, y) the lower-left corner of cell (0, 0); cells outside the grid
 * are free.  Each environment uses at most one map and may use none; maps never move and are not obstacles (the obstacle rows of
 * nb_world_read_state do not change; by default reactive obstacles do not see maps and moving obstacles pass over them, unless
 * nb_world_set_map_contact below makes an environment's map block its obstacles).
 *   maps (P) HOST; bits uint32 HOST: the maps back to back, each `height` rows of ceil(width/32) words, row j being y index j, bit
 *   (i mod 32) of word i/32 being cell (i, j) (padding bits 0); env_map (B) int32 HOST: each environment's map, -1 for none;
 *   window (0, 10] m, for the whole handle.
 *   scan    a beam also stops where it crosses from a free into an occupied cell or back (the first t > 0, corners count), with
 *           hit index O_b + K (after the obstacles and the robots, which win a tie) and velocity 0
 *   step    each robot's clearance is also bounded by m = min(window, its exact clearance to the occupied cells, each a square);
 *           m <= 0 sets collided
 * nb_world_set_maps comes after nb_world_set_scenes(_ex) and, if used, nb_world_set_fleet(_ex), which both drop the maps (a new
 * placement needs a new start check); behaviours are untouched.  It uploads the maps, checks them against the robots the handle
 * has placed, and synchronises the device.  A world without maps launches the same kernels as before.
 * Checks (NB_ERR_INVALID, naming the map, environment or robot): P in 1..max_envs; width and height in 1..8192; a finite origin;
 * a finite resolution >= 0.01; no padding bit set; env_map entries in -1..P-1; window in (0, 10]; no start body that overlaps or
 * touches an occupied cell of its environment's map (SAT, each robot's own polygon).  nb_world_check_maps performs them on the
 * host without a handle or a device; its first arguments are those of nb_world_check_fleet_ex (robots NULL: the maps are checked
 * without the start bodies).  Maps too large for the device fail with NB_ERR_CUDA and leave the handle usable, without maps. */
typedef struct nb_world_map {
  int32_t width, height;           /* cells, 1..8192 each */
  double origin[2];                /* the lower-left corner of cell (0, 0) */
  double resolution;               /* the side of a cell (m), >= 0.01 */
} nb_world_map;

int nb_world_check_maps(const nb_world_config* cfg, int32_t T, const nb_world_robot_type* types, int32_t B, int32_t K, const double* robots,
                        const int32_t* robot_type, int32_t P, const nb_world_map* maps, const uint32_t* bits, const int32_t* env_map,
                        double window);
int nb_world_set_maps(nb_world_t* w, int32_t P, const nb_world_map* maps, const uint32_t* bits, const int32_t* env_map, double window);

/* Obstacles in occupancy maps (semantics in csrc/world_kernel.cuh and csrc/world_rvo_kernel.cuh): flags (B) int32 HOST, 1 where an
 * environment's map blocks its obstacles, 0 (the default, and every environment without this call) where obstacles pass over it.
 * Where it is 1:
 *   contact   an obstacle touches the map when its footprint has clearance <= 0 to an occupied cell (a circle: its centre's distance
 *             to the cell minus r; a convex polygon or an outline: its exact clearance to the cell as a square)
 *   move      every moving obstacle (constant or reactive) takes, after its move and rectangle mirror (c', v') from (c, v), the first
 *             of A (c'x, c'y) with (v'x, v'y), B (c'x, cy) with (v'x, -v'y), C (cx, c'y) with (-v'x, v'y), D (cx, cy) with
 *             (-v'x, -v'y) whose footprint does not touch the map; D always (the start is clear), so no moving obstacle ever touches
 *             the map.  A step in which A is rejected is a bounce (nb_world_read_map_contact counts them per obstacle).
 *   reactive  the choice of the velocity is unchanged (the map is not a neighbour and has no cone).  A wander goal is accepted when the
 *             footprint at the goal does not touch the map and the segment from the centre to the goal keeps a distance > the
 *             obstacle's circumradius from every occupied cell; a rejected draw uses up its number; at most 16 draws per obstacle and
 *             step, and when all fail the obstacle parks for the step (goal = its centre) and draws the following numbers at the next
 *             step.  An obstacle whose move bounced treats its goal as reached at its next step.  A wandering obstacle without an
 *             explicit goal is set back to goal = its centre and draw 0 by this call, so that its first goal is drawn on the device
 *             through the test; explicit goals and goals without wander are not tested.
 * nb_world_set_map_contact comes after nb_world_set_maps (and nb_world_set_behaviors); nb_world_set_scenes(_ex),
 * nb_world_set_fleet(_ex), nb_world_set_behaviors and nb_world_set_maps drop it, and it leaves episode mode (nb_world_set_episodes
 * comes after it: then scene s's flag holds for its obstacles in whatever slot runs it).  It zeroes the bounce counts and
 * synchronises the device.  Without a flag set the kernels launched are those of a world without this call.
 * Checks (NB_ERR_INVALID, naming the environment and obstacle): every flag is 0 or 1, and 1 only where the environment has a map;
 * every moving obstacle (v != 0, or reactive) of a blocking environment starts with clearance > 0 to the map, and its top speed times
 * step_time (|v| for a constant obstacle, sqrt(vxmax^2 + vymax^2) for a reactive one) is below the map's resolution, so that it cannot
 * jump through a wall at least one cell thick.  Static obstacles may overlap walls.  Occupied cells that meet only at a corner can
 * still be crossed by a footprint smaller than one step.  nb_world_check_map_contact performs them on the host without a handle or a
 * device (behaviors NULL: every obstacle keeps its constant velocity).
 * nb_world_read_map_contact enqueues a device-to-device copy of the O per-obstacle bounce counts on `stream` and does not synchronise.
 * Not modelled: walls as RVO neighbours (ORCA lines), moving maps, swept or continuous collision; obstacle-obstacle contact is the
 * separate nb_world_set_obstacle_contact below. */
int nb_world_check_map_contact(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obstacles, const int32_t* vert_begin,
                               const double* vertices, const double* envs, const int32_t* obs_kind, const double* behaviors, int32_t P,
                               const nb_world_map* maps, const uint32_t* bits, const int32_t* env_map, const int32_t* flags);
int nb_world_set_map_contact(nb_world_t* w, int32_t B, const int32_t* flags);
int nb_world_read_map_contact(nb_world_t* w, int32_t O, int32_t* bounces, void* stream);

/* Obstacle contact (semantics in csrc/world_contact_kernel.cuh): flags (B) int32 HOST, 1 where an environment's obstacles block each
 * other, 0 (the default, and every environment without this call) where they pass through each other.  Where it is 1:
 *   touch     two footprints touch when their clearance is <= 0: circle-circle by centre distance - (r_i + r_j); circle-convex by the
 *             circle test of the robot clearance; circle-outline by even-odd or centre-edge distance <= r; convex-convex and
 *             convex-outline by the robot clearance tests; outline-outline when two edges meet or vertex 0 of either lies inside the
 *             other.  A pair is tested only when the boxes of the two footprints, each widened by 1e-6 m, meet.  The test is symmetric
 *             bit for bit.
 *   move      the obstacles move in ascending row order.  Every moving obstacle (v != 0 after the rvo kernel) takes, after its move and
 *             rectangle mirror (c', v') from (c, v), the first of A (c'x, c'y) with (v'x, v'y), B (c'x, cy) with (v'x, -v'y), C
 *             (cx, c'y) with (-v'x, v'y), D (cx, cy) with (-v'x, -v'y) whose footprint touches no other obstacle of its environment (the
 *             earlier rows at their new centres, the later rows at their old ones, static obstacles included) and, where the map
 *             blocks obstacles, not the map either.  D always (the start is clear), so no moving obstacle ever touches another
 *             obstacle.  A step whose A touches another obstacle is an obstacle bounce (nb_world_read_obstacle_contact counts them per
 *             obstacle); the map's bounce count and a reactive obstacle's reaction to it keep their meaning (A touched the map).
 *             Reactive obstacles choose their velocity as before.  Robots do not block obstacles (an obstacle may still move into a
 *             robot, which then collides).
 * nb_world_set_obstacle_contact comes after nb_world_set_scenes(_ex), nb_world_set_behaviors, nb_world_set_fleet(_ex),
 * nb_world_set_maps and nb_world_set_map_contact, which all drop it; it leaves episode mode (nb_world_set_episodes comes after it:
 * then scene s's flag and bounce counts hold for its obstacle rows in whatever slot runs it).  It zeroes the bounce counts and
 * synchronises the device.  With a flag set nb_world_step launches one more kernel (the obstacles move there, one warp per
 * environment); without one the kernels launched are those of a world without this call.
 * Checks (NB_ERR_INVALID, naming the environment and obstacle rows): B is the handle's environment count; every flag is 0 or 1; no
 * obstacle that can move (v != 0, or reactive) of an environment with the flag set starts touching another obstacle of it, by the
 * same test on the host.  Static obstacles may overlap each other.  nb_world_check_obstacle_contact performs them on the host
 * without a handle or a device (behaviors NULL: every obstacle keeps its constant velocity).
 * nb_world_read_obstacle_contact enqueues a device-to-device copy of the O per-obstacle bounce counts on `stream` and does not
 * synchronise.
 * Limits: no swept test (a step longer than the thinner of two footprints can pass through it; dyna_obs's circles move at most
 * 0.05 m per step at step_time 0.1 s), no contact with robots, no momentum or elastic response, and earlier rows move first. */
int nb_world_check_obstacle_contact(const nb_world_config* cfg, int32_t B, const int32_t* obs_begin, const double* obstacles, const int32_t* vert_begin,
                                    const double* vertices, const double* envs, const int32_t* obs_kind, const double* behaviors, const int32_t* flags);
int nb_world_set_obstacle_contact(nb_world_t* w, int32_t B, const int32_t* flags);
int nb_world_read_obstacle_contact(nb_world_t* w, int32_t O, int32_t* bounces, void* stream);

/* Continuous episodes (semantics in csrc/world_episode_kernel.cuh): a bank of S scenes runs through `slots` slots, and a slot starts
 * the next unstarted scene on the device when its episode ends.  The bank is uploaded as a world of B = S environments
 * (nb_world_set_scenes(_ex), then optionally nb_world_set_behaviors, nb_world_set_fleet(_ex), nb_world_set_maps; S <= max_envs, one
 * K for every scene, and robot k of the same type in every scene).  nb_world_set_episodes(w, slots, max_steps) then switches the
 * handle to episode mode: slot b starts on scene b; every per-scene array stays where the set calls put it, a slot only names the
 * scene it runs (scene_of), and every scene runs once.  It allocates the slot and result arrays and synchronises the device.
 *   nb_world_scan, nb_world_step, nb_world_read_state take N = slots*K; their per-robot arrays are slot rows (robot k of slot b at
 *           row b*K + k): ranges, velocity, hit, action, collided / arrived / clearance, states.  Reactive obstacles draw their goals
 *           keyed by the scene index, as environment s of a plain world does.  nb_world_read_state with N = S*K reads the scenes' own
 *           rows instead (a scene's final state once its episode has ended: nothing touches its rows again); obstacles are the S
 *           scenes' rows either way.  nb_world_read_behaviors takes B = S.
 *   end     after step t of a scene (t = 1 at its first step in its slot) its episode ends when every robot of the scene has collided
 *           or arrived (reason 1, "flags") or when t == max_steps (reason 2, "timeout"; flags win a tie at the same step).
 *   next    after every nb_world_step a kernel records the ended episodes' results and hands out the next unstarted scenes: the slots
 *           whose episode ended in this step, in ascending slot order, take the next scenes in ascending scene order.  When the bank
 *           is exhausted a slot goes idle: its scene is frozen (no integration, no obstacle motion, no flag or result changes; its
 *           scan is that scene's scan, its step outputs are the frozen flags and clearance +inf).  reset[b] = 1 for a slot that has
 *           just taken a new scene (every slot after nb_world_set_episodes), else 0.  In episode mode nb_world_step launches one
 *           more kernel than a plain world (the advance kernel), and nb_world_read_state of slot rows launches one gather kernel where
 *           a plain world copies.  Nothing synchronises the host.
 * nb_world_read_episodes (B = S) reads, DEVICE outputs, any may be NULL, enqueued on `stream`: per robot of a scene (S*K rows)
 * collided, arrived (the flags at the episode's end), arrive_step (the step of arrival, -1 if none: rollout's steps_to_arrive) and
 * min_clearance (the smallest clearance over the episode's steps), all 0 / -1 / +inf until it has ended; per scene (S) end_step
 * (0 until it has ended), reason (0 until then, 1 flags, 2 timeout) and slot (the slot that ran it, -1 until it has started); per
 * slot scene_of and reset (slots); finished (1): the episodes ended so far.
 * nb_world_set_scenes(_ex), nb_world_set_fleet(_ex), nb_world_set_behaviors and nb_world_set_maps leave episode mode.
 * Checks (NB_ERR_INVALID, naming the scene and robot): S in 1..max_envs, K in 1..16, slots in 1..S, max_steps >= 1, robot_type (S*K,
 * HOST, or NULL: every robot type 0) giving robot k the type of robot k of scene 0 in every scene.  nb_world_check_episodes performs
 * them on the host without a handle or a device.
 * Limits: one max_steps per handle; no multi-GPU episode runs; the bank must fit max_envs and device memory. */
int nb_world_check_episodes(const nb_world_config* cfg, int32_t S, int32_t K, const int32_t* robot_type, int32_t slots, int32_t max_steps);
int nb_world_set_episodes(nb_world_t* w, int32_t slots, int32_t max_steps);
int nb_world_read_episodes(nb_world_t* w, int32_t S, int32_t* collided, int32_t* arrived, int32_t* arrive_step, float* min_clearance,
                           int32_t* end_step, int32_t* reason, int32_t* slot, int32_t* scene_of, int32_t* reset, int32_t* finished,
                           void* stream);

/* Actuation limits and noise (semantics in csrc/world_kernel.cuh; this project's reading of IR-SIM's vel_min / vel_max / acce and
 * its motion and lidar `noise` switches, not a claim of parity).  Both are off until these calls; a handle without them launches the
 * kernels of a world without them.
 *   nb_world_set_actuation: per_type (num_types, HOST) one row per robot type of the handle (type 0 the config's robot, then the
 *           types of nb_world_set_fleet_ex), in the action's own convention (diff (v, omega), acker (v, steering), omni (vx, vy)):
 *           vel_min / vel_max (-inf / +inf: no bound), acce (+inf: no rate limit), alpha (0: no motion noise).  In a step robot n
 *           with action a takes, per component, c = min(max(a, max(vel_min, cmd_prev - acce dt)), min(vel_max, cmd_prev + acce dt)),
 *           stores cmd_prev = c, and integrates u = c + (s0 z0, s1 z1) with s0 = sqrt(alpha0 c0^2 + alpha1 c1^2), s1 = sqrt(alpha2 c0^2
 *           + alpha3 c1^2) and standard normal z from the motion stream (`seed`); the scan's velocity of the robot is that of u.  A
 *           collided robot stays frozen and its cmd_prev becomes 0.  Reactive obstacles still see the action as given.  From this
 *           call on nb_world_step launches the step's actuation variant.
 *           Checks (NB_ERR_INVALID, naming the type and component): num_types is the handle's type count, no NaN, vel_min <= vel_max
 *           (vel_min < +inf, vel_max > -inf), acce > 0, alpha finite and >= 0, an acker type's finite steering limits in (-pi/2, pi/2).
 *   nb_world_set_lidar_noise: a beam that hits something reports clamp(t + range_std z, range_min, range_max) (FP64, then the float
 *           cast); a miss (range_max), the hit index and the velocity are unchanged; z from the lidar stream (`seed`).  range_std 0
 *           turns it off.  Checks (NB_ERR_INVALID): range_std finite and >= 0, range_min in [0, range_max).
 *   streams z is keyed by (seed, environment e, robot k within it, the scene's step n, component or beam j), with a domain tag per
 *           use (motion, lidar), independent of the reactive obstacles' goal draws.  n counts the nb_world_step calls since the
 *           robots were placed in a plain world, and is the slot's episode step in episode mode (e the scene there); the first scan
 *           and step use n = 0.  So environment e's noise does not depend on B, two scans without a step between them are equal, and
 *           an episode is bitwise the plain run of its scene.
 * The settings are kept by nb_world_set_scenes(_ex), nb_world_set_fleet(_ex) and nb_world_set_episodes, which zero cmd_prev (so
 * does a slot taking a new scene); types past num_types (a later fleet with more types) take the defaults.
 * nb_world_read_commands enqueues on `stream` a device-to-device copy of cmd_prev (N, 2) float64, N = B*K (S*K, the scenes' rows, in
 * episode mode), without synchronising. */
typedef struct nb_world_actuation {
  double vel_min[2], vel_max[2], acce[2], alpha[4];
} nb_world_actuation;

int nb_world_set_actuation(nb_world_t* w, int32_t num_types, const nb_world_actuation* per_type, uint64_t seed);
int nb_world_set_lidar_noise(nb_world_t* w, double range_min, double range_std, uint64_t seed);
int nb_world_read_commands(nb_world_t* w, int32_t N, double* cmd_prev, void* stream);

/* ---- DUNE training on the device (SURVEY 8f "next" row 4) ------------------------------------------------------------ */

/* DUNETrain.generate_data_set / prob_solve (neupan/blocks/dune_train.py:100-140): labels of n sampled points -- the solution of the
 * cone program (10) max mu'(G p - h) s.t. |G' mu| <= 1, mu >= 0, in closed form (the reference calls cvxpy/ECOS once per point).
 * HOST: G (E x 2), h (E).  DEVICE: points (n,2) float64 in, points_f32 (n,2), mu (n,E), dist (n) float32 out. */
int nb_dune_labels(int32_t edge_dim, const float* G, const float* h, int64_t n, const double* points,
                   float* points_f32, float* mu, float* dist, void* stream);

typedef struct nb_dune_train nb_dune_train_t; /* owns the parameters being trained and Adam's moments */

/* DUNETrain.__init__ (dune_train.py:61-80): weights (HOST, packed like nb_pan_create's) are the initial parameters; the optimiser is
 * Adam(lr, betas (0.9, 0.999), eps 1e-8, weight_decay 1e-4) as at :72. */
int nb_dune_train_create(int32_t edge_dim, const float* G, const float* h, const float* weights, int64_t n_weights,
                         int32_t device, nb_dune_train_t** out);
int nb_dune_train_destroy(nb_dune_train_t* t);

/* DUNETrain.train_one_epoch (dune_train.py:281-333): one pass over n labelled points (DEVICE: pts (n,2), mu (n,E), dist (n)) in
 * batches of batch_size <= 256 taken in order (DataLoader without shuffling), loss MSE(mu) + MSE(distance) + MSE(fa) + MSE(fb) with
 * the rotation angle thetas[b] (HOST, one per batch; the reference draws np.random.uniform(0, 2 pi) per batch, :351) and, unless
 * `validate`, one Adam step per batch.  losses (HOST, 4 doubles) = the four terms averaged over the batches.  Synchronises `stream`. */
int nb_dune_train_epoch(nb_dune_train_t* t, const float* pts, const float* mu, const float* dist, int64_t n, int32_t batch_size,
                        const float* thetas, float lr, int32_t validate, double* losses, void* stream);

/* The current parameters (HOST, packed): torch.save(model.state_dict()) at :247-252 after unpacking. */
int nb_dune_train_get_weights(nb_dune_train_t* t, float* weights);

/* Number of kernel launches issued by this library since load (bench.py's gpu_launches). */
int64_t nb_launch_count(void);
/* Number of device allocations the library holds right now, over every handle of the process (a handle that is destroyed gives
 * back all of its own). */
int64_t nb_buffer_count(void);
const char* nb_last_error(void);
int nb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* NEUPAN_B200_H */
