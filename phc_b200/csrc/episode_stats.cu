// Episode statistics of the rollout (phc/learning/amp_agent.py:358-369 with rl_games 1.1.4's AverageMeter), one launch per step,
// captured in the rollout graph.  The reference indexes the done envs on the host (`dones.nonzero()`, a sync every step) and folds
// their returns and lengths into two AverageMeters; here one block walks all envs:
//   v_r = cur_r + r, v_l = cur_l + 1                 (this step's running return and length)
//   the done envs' v_r, v_l are summed (fp64) and counted
//   cur_r = v_r * (1 - done), cur_l = v_l * (1 - done)   (the same fp32 operations as `add_(r).mul_(1 - done.float())`)
// and thread 0 applies AverageMeter.update with the mean over ALL k done envs:
//   size = min(k, max_size); old = min(max_size - size, current_size)
//   mean = (mean * old + new_mean * size) / (old + size); current_size = old + size
// One block, a fixed per-thread stride, fixed-order shuffles and warps added in order: no atomics, bit-identical from run to run.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/phc_b200.h"

namespace phc {
namespace epstats {

constexpr int kThreads = 512;

__device__ __forceinline__ double wsum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int wsum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// mean[2] / size[2]: the game_rewards and game_lengths meters (fp32 mean, int32 current_size)
__global__ void __launch_bounds__(kThreads)
episode_stats_kernel(const float* __restrict__ rewards, const int64_t* __restrict__ dones, int64_t n, float* __restrict__ cur_r,
                     float* __restrict__ cur_l, float* __restrict__ mean, int32_t* __restrict__ size, int32_t max_size) {
  __shared__ double w_r[kThreads / 32], w_l[kThreads / 32];
  __shared__ int w_k[kThreads / 32];
  double sr = 0.0, sl = 0.0;
  int k = 0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const int64_t d = dones[i];
    const float nd = 1.0f - (float)d;
    const float vr = cur_r[i] + rewards[i];
    const float vl = cur_l[i] + 1.0f;
    if (d != 0) {
      sr += (double)vr;
      sl += (double)vl;
      ++k;
    }
    cur_r[i] = vr * nd;
    cur_l[i] = vl * nd;
  }
  sr = wsum(sr);
  sl = wsum(sl);
  k = wsum_i(k);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) {
    w_r[w] = sr;
    w_l[w] = sl;
    w_k[w] = k;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double tr = 0.0, tl = 0.0;
  int tk = 0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) {
    tr += w_r[i];
    tl += w_l[i];
    tk += w_k[i];
  }
  if (tk == 0) return;
  const int s = tk < max_size ? tk : max_size;
  const float new_mean[2] = {(float)(tr / tk), (float)(tl / tk)};
  for (int m = 0; m < 2; ++m) {
    const int old = (max_size - s) < size[m] ? (max_size - s) : size[m];
    // fp32 as torch evaluates `(mean * old + new_mean * size) / size_sum`: two rounded products, no contraction
    mean[m] = (__fmul_rn(mean[m], (float)old) + __fmul_rn(new_mean[m], (float)s)) / (float)(old + s);
    size[m] = old + s;
  }
}

}  // namespace epstats
}  // namespace phc

extern "C" void phc_set_error(const char* msg);
extern "C" int phc_check_cuda(cudaError_t e, const char* what);
extern "C" void phc_count_launches(int n);

extern "C" int phc_episode_stats(const float* rewards, const int64_t* dones, int64_t n, float* cur_r, float* cur_l, float* meter_mean,
                                 int32_t* meter_size, int32_t games_to_track, void* stream) {
  using namespace phc::epstats;
  if (n <= 0) { phc_set_error("phc_episode_stats: n <= 0"); return PHC_ERR_INVALID_ARG; }
  if (games_to_track < 1) { phc_set_error("phc_episode_stats: games_to_track < 1"); return PHC_ERR_INVALID_ARG; }
  if (!rewards || !dones || !cur_r || !cur_l || !meter_mean || !meter_size) {
    phc_set_error("phc_episode_stats: a required pointer is NULL"); return PHC_ERR_INVALID_ARG;
  }
  episode_stats_kernel<<<1, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(rewards, dones, n, cur_r, cur_l, meter_mean, meter_size,
                                                                              games_to_track);
  phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "episode_stats_kernel launch");
}
