// Shared definitions of the PAN hot-path kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nb {

constexpr int kHidden = 32;   // ObsPointNet hidden width (obs_point_net.py:29)
constexpr int kMaxEdges = 8;  // largest supported E = G.shape[0]
constexpr int kCandMax = 32;  // candidates per (environment, step) item kept by the DUNE screening pass (dune_screen_kernel.cuh)

// offsets (in floats) into the packed checkpoint, state_dict key order
// MLP.{0,1,3,5,6,8,10,11,13}.{weight,bias} (obs_point_net.py:31-46); all multiples of 32.
struct WeightLayout {
  static constexpr int W0 = 0, B0 = 64, G1 = 96, BE1 = 128;
  static constexpr int W3 = 160, B3 = 1184, W5 = 1216, B5 = 2240, G6 = 2272, BE6 = 2304;
  static constexpr int W8 = 2336, B8 = 3360, W10 = 3392, B10 = 4416, G11 = 4448, BE11 = 4480;
  static constexpr int W13 = 4512;
  __host__ __device__ static constexpr int b13(int E) { return 4512 + 32 * E; }
  __host__ __device__ static constexpr int count(int E) { return 4512 + 33 * E; }
};

// robot polygon G x <= h (gen_inequal_from_vertex), float32 as np_to_tensor makes it (dune.py:45-46)
struct Geometry {
  float G[kMaxEdges][2];
  float h[kMaxEdges];
  int E;
};

}  // namespace nb
