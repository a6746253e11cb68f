// Definitions shared by the DUNE kernels (dune_tc_kernel.cuh, dune_screen_kernel.cuh, dune_screen_mma_kernel.cuh,
// dune_table_kernel.cuh): the launch parameters, the distance-table lookup, the sort key and the point flow.
//
// The kernels replace, for a whole batch of environments and all T+1 horizon steps in one pipeline:
//   PAN.generate_point_flow / point_state_transform   neupan/blocks/pan.py:150-212
//   ObsPointNet.forward                                neupan/blocks/obs_point_net.py:31-49
//   DUNE.forward / cal_objective_distance              neupan/blocks/dune.py:58-127
// Only the first M = nrmp_max_num sorted columns are ever consumed downstream
// (nrmp.py:136-138,254-256; pan.py:234-237), so the full argsort of dune.py:100 is replaced by a
// deterministic top-M selection (ascending distance, ties -> lower point index).
#pragma once
#include <vector>

#include "common.cuh"

namespace nb {

struct DuneParams {
  const float* weights;       // packed checkpoint (device)
  const float* nom_s;         // (B,3,T+1)
  const float* points;        // (B,2,N)
  const float* velocities;    // (B,2,N) or nullptr
  const int32_t* num_points;  // (B) or nullptr
  const int32_t* active;      // (B) or nullptr: env skipped when 0
  float* sel_mu;              // (B,T+1,M,E)
  float* sel_lam;             // (B,T+1,M,2)
  float* sel_pts;             // (B,T+1,M,2)
  float* sel_dist;            // (B,T+1,M)
  int32_t* sel_count;         // (B)
  float* min_dist;            // (B) or nullptr
  int B, N, T, M;
  float dt;
  Geometry geo;
  // screening (NB_OPT_DUNE_KERNEL = 4, dune_screen_kernel.cuh): candidate lists written by dune_screen_kernel, consumed by
  // dune_refine_kernel; all nullptr / 0 in the other variants
  int32_t* cand_idx;        // (B (T+1), 32) point indices
  int32_t* cand_cnt;        // (B (T+1)): candidates of the item; -1 = evaluate the item exactly; 0 = nothing to do
  float* cand_dt;           // (B (T+1), 32) screened distance of each candidate (NaN: not screened) -- statistics only
  float* cand_rad;          // (B (T+1), 32) the error radius the screen assumed for each candidate (checked by the refine kernel)
  unsigned* screen_stats;   // [0] max |d~ - d| / sum|t| over candidates (float bits), [1] items sent to the exact kernel, [2] candidates, [3] items screened
  float c_mu;               // bound on |mu~_e - mu_e| of the screening network
  // distance table of the mma.sync screen (dune_table_kernel.cuh); tab_cell == nullptr: every point runs the screening network
  const float4* tab_cell;   // (n, n) cells, row iy: {d(ix, iy), d(ix+1, iy), d(ix, iy+1), d(ix+1, iy+1)} at the cell's corners
  const float* tab_rad;     // (n, n) the cell's error radius
  int tab_n;                // cells per side
  float tab_half, tab_inv_h;  // the table covers [-tab_half, tab_half]^2 of the robot frame with cells of 1 / tab_inv_h metres
  // coarse bound table of dune_screen_warp_kernel (dune_table_kernel.cuh): coarse cell (ix >> kCoarseLog, iy >> kCoarseLog) of fine cell
  // (ix, iy) holds {LB, UB} as fp16 (low, high half) with LB <= table_bilerp - rad and UB >= table_bilerp + rad of every point of its fine
  // cells; nullptr: every item takes the one-level table path (NB_SCREEN_COARSE=0)
  const uint32_t* tab_coarse;
  int tab_cn;               // coarse cells per side
  unsigned* coarse_stats;   // [0] survivors of the coarse pass, [1] table items that took the one-level path (nb_pan_read_screen_coarse)
  int32_t* flag_list;       // (B (T+1)) the items with cand_cnt == -1, in the order the screen kernel met them
  int32_t* flag_count;      // (3) [0] their number, [1] / [2] the lengths of the two refine lists; zeroed by the launcher before the screen kernel
  int32_t* refine_list;     // (2 B (T+1)) work lists of dune_refine_kernel, appended by the screen kernels: [0, B (T+1)) the items with 1..16
                            // candidates (two of them share a warp), [B (T+1), 2 B (T+1)) those with 17..32 (one warp each)
  int only_flagged;         // exact kernel: process only the items of flag_list
  int skip_t0;              // screen kernels: step-0 items are skipped (cand_cnt = 0) and keep the outputs of the previous launch -- set by
                            // nb_pan_forward for PAN iterations k > 0: nom_s[:, 0] is the fixed initial state (robot.py:234; the NRMP kernel
                            // copies the column bit for bit), so item (b, 0) has the same inputs and the same result in every iteration
  int screen_mma;           // launcher hint (NB_OPT_DUNE_SCREEN_MMA): 1 = screening pass on mma.sync (dune_screen_mma_kernel.cuh) where N <= 1024
  int calibrate;            // screen kernel: items with N <= 32 are NOT short-cut: all their points become candidates with their screened
                            // distance, so that the refine kernel's statistics compare the two networks on every point (nb_pan calibration)
};

// bilinear interpolation inside a table cell: c = the corner values {d00, d10, d01, d11}, (a, b) in [0, 1]^2 the position in the
// cell.  The table build measures the cell's error radius with this same function.
__device__ __forceinline__ float table_bilerp(const float4& c, float a, float b) {
  const float d0 = fmaf(a, c.y - c.x, c.x), d1 = fmaf(a, c.w - c.z, c.z);
  return fmaf(b, d1 - d0, d0);
}

constexpr int kCoarseLog = 4;  // a coarse bound cell covers 16 x 16 fine cells of the distance table

// the table cell (ix, iy) of the robot-frame point (x, y) and the point's position (a, b) in it; false when the point lies outside the table
__device__ __forceinline__ bool table_cell_xy(const DuneParams& prm, float x, float y, int& ix, int& iy, float& a, float& b) {
  const float fx = (x + prm.tab_half) * prm.tab_inv_h, fy = (y + prm.tab_half) * prm.tab_inv_h, nf = (float)prm.tab_n;
  if (!(fx >= 0.f && fx < nf && fy >= 0.f && fy < nf)) return false;  // NaN coordinates are outside as well
  ix = (int)fx;
  iy = (int)fy;
  a = fx - (float)ix;
  b = fy - (float)iy;
  return true;
}

// the same as table_cell_xy with the cell as one index c = iy n + ix
__device__ __forceinline__ bool table_cell(const DuneParams& prm, float x, float y, int& c, float& a, float& b) {
  int ix, iy;
  if (!table_cell_xy(prm, x, y, ix, iy, a, b)) return false;
  c = iy * prm.tab_n + ix;
  return true;
}

// screened distance d and error radius r of the robot-frame point (x, y) from the table; false when the point lies outside it
__device__ __forceinline__ bool table_lookup(const DuneParams& prm, float x, float y, float& d, float& r) {
  int c;
  float a, b;
  if (!table_cell(prm, x, y, c, a, b)) return false;
  d = table_bilerp(__ldg(prm.tab_cell + c), a, b);
  r = __ldg(prm.tab_rad + c);
  return true;
}

__device__ __forceinline__ uint32_t orderable(float d) {
  if (d != d) return 0xFFFFFFFFu;  // NaN sorts last
  uint32_t u = __float_as_uint(d);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// p_t = p + t*(v*dt) with the reference's rounding sequence (pan.py:182), no FMA contraction
__device__ __forceinline__ float flow(float p, float v, float dt, int t) {
  return __fadd_rn(p, __fmul_rn((float)t, __fmul_rn(v, dt)));
}

// dune_tc.cu: the operand images of the warpgroup kernels (screen = true: of the screening network) from a packed checkpoint, and the
// launch of the exact DUNE pass (screen = false) or of the screening pipeline (true); errors are reported through nb::fail
int build_tc_image(const float* w, int E, std::vector<unsigned char>& out, bool screen);
int launch_dune_tc(const DuneParams& prm, const unsigned char* d_image, const unsigned char* d_screen_image, int image_flags, bool screen, int sm_count,
                   int max_smem_optin, cudaStream_t st);

}  // namespace nb
