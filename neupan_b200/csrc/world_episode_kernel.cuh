// Continuous episodes in the batched world (nb_world_set_episodes): a bank of S scenes, uploaded like any B = S world, runs through
// `slots` slots.  Slot b runs scene scene_of[b]; the scan, rvo and step kernels take the scene through scene_of (their kEp
// instantiations, world_kernel.cuh).  After every nb_world_step, world_advance_kernel ends episodes and hands out the next scenes:
//
//   end      a live slot's scene has taken step t (t counts from 1 at its first step in the slot); its episode ends when every robot
//            of the scene has collided or arrived ("flags", reason 1) or when t == max_steps ("timeout", reason 2; flags win a tie).
//            The results are recorded then: per robot the sticky flags, the step of arrival (-1 if none: rollout's steps_to_arrive)
//            and the smallest clearance over the episode's steps (accumulated every step), per scene the end step and the reason.
//   next     the slots whose episode ended in this step, in ascending slot order, take the next unstarted scenes in ascending scene
//            order (one block-wide exclusive scan over the slots); a slot for which none is left goes idle: its scene is frozen and
//            no kernel touches its rows again.  reset[b] = 1 for a slot that has just taken a new scene, else 0.  With actuation
//            set (nb_world_set_actuation) the new scene's cmd_prev rows are zeroed.
//
// Every scene runs once, so nothing needs restoring at a reset: a scene's own rows hold its start until its slot takes it and its
// final state after its episode.
#pragma once
#include <cstdint>

namespace nb {

constexpr int kWorldAdvanceThreads = 1024;

struct WorldEpisodeParams {
  int S, slots, K, max_steps;
  int32_t* scene_of;        // (slots)
  int32_t* live;            // (slots) 0: idle
  int32_t* reset;           // (slots) 1: took a new scene in this step
  int32_t* t;               // (slots) steps of the current episode
  int32_t* next;            // (1) the next unstarted scene (may pass S)
  int32_t* finished;        // (1) episodes ended so far
  const int32_t* collided;  // (S K) the scenes' sticky flags
  const int32_t* arrived;
  const float* clear;       // (slots K) this step's clearances (world_step_kernel<., true>)
  int32_t* r_col;           // (S K) results per robot of a scene
  int32_t* r_arr;
  int32_t* r_astep;
  float* r_minclr;
  int32_t* r_end;           // (S) results per scene: end step (0 while running), reason (0 while running), the slot that ran it
  int32_t* r_reason;
  int32_t* r_slot;
  double* cmd;              // (S K, 2) cmd_prev of the scenes' robots (nb_world_set_actuation), or NULL
};

// One CTA: thread i takes the contiguous slots [i c, (i + 1) c), c = ceil(slots / blockDim), so that ascending threads are
// ascending slots.  Pass 1 records the ended episodes and marks them in reset[]; the scan ranks them; pass 2 hands out the scenes.
__global__ void __launch_bounds__(kWorldAdvanceThreads) world_advance_kernel(const WorldEpisodeParams ep) {
  __shared__ int s_warp[kWorldAdvanceThreads / 32];
  const int c = (ep.slots + blockDim.x - 1) / blockDim.x;
  const int lo = min((int)threadIdx.x * c, ep.slots), hi = min(lo + c, ep.slots);
  const int K = ep.K;
  int ended = 0;
  for (int b = lo; b < hi; ++b) {
    int end = 0;
    if (ep.live[b] != 0) {
      const int e = ep.scene_of[b], t = ep.t[b] + 1;
      ep.t[b] = t;
      bool done = true;
      for (int k = 0; k < K; ++k) {
        const size_t n = (size_t)e * K + k;
        const int col = ep.collided[n], arr = ep.arrived[n];
        if (arr != 0 && ep.r_astep[n] < 0) ep.r_astep[n] = t;
        ep.r_minclr[n] = fminf(ep.r_minclr[n], ep.clear[(size_t)b * K + k]);
        done = done && (col != 0 || arr != 0);
      }
      if (done || t == ep.max_steps) {
        for (int k = 0; k < K; ++k) {
          const size_t n = (size_t)e * K + k;
          ep.r_col[n] = ep.collided[n];
          ep.r_arr[n] = ep.arrived[n];
        }
        ep.r_end[e] = t;
        ep.r_reason[e] = done ? 1 : 2;
        end = 1;
        ++ended;
      }
    }
    ep.reset[b] = end;
  }
  // exclusive scan of the per-thread counts: warp shuffles, then the warp totals
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int base = *ep.next;  // every thread reads it before thread 0 moves it on (the barriers below)
  int incl = ended;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) s_warp[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    const int nwarps = blockDim.x >> 5;
    int v = lane < nwarps ? s_warp[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, v, d);
      if (lane >= d) v += u;
    }
    if (lane < nwarps) s_warp[lane] = v;  // inclusive totals of warps 0 .. lane
  }
  __syncthreads();
  int rank = (wid > 0 ? s_warp[wid - 1] : 0) + incl - ended;
  for (int b = lo; b < hi; ++b) {
    if (ep.reset[b] == 0) continue;
    const int s = base + rank++;
    if (s < ep.S) {
      ep.scene_of[b] = s;
      ep.t[b] = 0;
      ep.r_slot[s] = b;
      if (ep.cmd)  // the new scene's robots start from a zero command
        for (int k = 0; k < 2 * K; ++k) ep.cmd[2 * (size_t)s * K + k] = 0.0;
    } else {
      ep.live[b] = 0;
      ep.reset[b] = 0;
    }
  }
  if (threadIdx.x == 0) {
    const int total = s_warp[(blockDim.x >> 5) - 1];
    *ep.next = base + total;
    *ep.finished += total;
  }
}

// nb_world_read_state of the slot rows: row q = b K + k of each output from scene row scene_of[b] K + k (one thread per row)
__global__ void __launch_bounds__(256) world_gather_kernel(int slots, int K, const int32_t* __restrict__ scene_of, const double* __restrict__ states,
                                                          const int32_t* __restrict__ collided, const int32_t* __restrict__ arrived,
                                                          double* __restrict__ out_states, int32_t* __restrict__ out_collided,
                                                          int32_t* __restrict__ out_arrived) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= slots * K) return;
  const int b = q / K;
  const size_t n = (size_t)scene_of[b] * K + (q - b * K);
  if (out_states) {
    out_states[3 * (size_t)q] = states[3 * n];
    out_states[3 * (size_t)q + 1] = states[3 * n + 1];
    out_states[3 * (size_t)q + 2] = states[3 * n + 2];
  }
  if (out_collided) out_collided[q] = collided[n];
  if (out_arrived) out_arrived[q] = arrived[n];
}

}  // namespace nb
