// PPO scalar kernels: GAE as a segmented warp scan, advantage normalisation.
// Reference: CommonAgent.discount_values (phc/learning/common_agent.py:493-505), returns = advs + values
// (phc/learning/amp_agent.py:384-385), CommonAgent._calc_advs (common_agent.py:589-599).
//
// GAE:  A_t = delta_t + c_t * A_{t+1},  delta_t = r_t + gamma*V'_t - V_t,  c_t = gamma*tau*(1 - done_t)
// is a first-order linear recurrence -> an associative scan over pairs (c, delta) with
//   (c_a, d_a) o (c_b, d_b) = (c_a*c_b, d_a + c_a*d_b);  done_t = 1 gives c_t = 0, i.e. a segment boundary.
// Data is time-major [T, N] (the reference's experience buffer), so a CTA takes 32 consecutive envs: warp w loads
// time row w coalesced (128 B), the tile is transposed through padded shared memory, warp e then scans env e along
// time with 5 shuffle steps, and rows are written back coalesced.  T > 32 is walked in chunks of 32 from the end
// with a carried A_{t+1}.  768 B per env per epoch: HBM/latency bound, one launch.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/phc_b200.h"

extern "C" void phc_set_error(const char* msg);
extern "C" int phc_check_cuda(cudaError_t e, const char* what);
extern "C" void phc_count_launches(int n);

namespace phc {

__global__ void __launch_bounds__(1024)
gae_kernel(const float* __restrict__ fdones, const float* __restrict__ values, const float* __restrict__ rewards,
           const float* __restrict__ next_values, int T, int64_t N, float gamma, float tau, float* __restrict__ advs,
           float* __restrict__ returns) {
  __shared__ float s_c[32][33], s_d[32][33], s_v[32][33];
  __shared__ float s_carry[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t env0 = (int64_t)blockIdx.x * 32;
  if (warp == 0) s_carry[lane] = 0.0f;
  const float gt = gamma * tau;
  for (int t_hi = T; t_hi > 0; t_hi -= 32) {
    const int t_lo = t_hi - 32 > 0 ? t_hi - 32 : 0;
    const int nt = t_hi - t_lo;
    __syncthreads();
    // phase 1: warp = time row (coalesced over envs)
    if (warp < nt) {
      const int t = t_lo + warp;
      const int64_t e = env0 + lane;
      float c = 0.f, d = 0.f, v = 0.f;
      if (e < N) {
        const int64_t i = (int64_t)t * N + e;
        v = values[i];
        const float nd = 1.0f - fdones[i];
        d = rewards[i] + gamma * next_values[i] - v;
        c = gt * nd;
      }
      s_c[warp][lane] = c; s_d[warp][lane] = d; s_v[warp][lane] = v;
    }
    __syncthreads();
    // phase 2: warp = env, lane = time inside the chunk; reverse (suffix) inclusive scan
    {
      float c = lane < nt ? s_c[lane][warp] : 0.0f;
      float d = lane < nt ? s_d[lane][warp] : 0.0f;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float c2 = __shfl_down_sync(0xffffffffu, c, o);
        const float d2 = __shfl_down_sync(0xffffffffu, d, o);
        if (lane + o < nt) { d = d + c * d2; c = c * c2; }
      }
      const float a = d + c * s_carry[warp];     // A_{t_hi} from the later chunk
      __syncwarp();
      if (lane < nt) s_d[lane][warp] = a;
      if (lane == 0) s_carry[warp] = a;          // A_{t_lo} feeds the next (earlier) chunk
    }
    __syncthreads();
    // phase 3: coalesced write-back
    if (warp < nt) {
      const int t = t_lo + warp;
      const int64_t e = env0 + lane;
      if (e < N) {
        const int64_t i = (int64_t)t * N + e;
        const float a = s_d[warp][lane];
        if (advs) advs[i] = a;
        if (returns) returns[i] = a + s_v[warp][lane];
      }
    }
  }
}

constexpr int kAdvBlock = 256;

// pass 1: adv = ret - val (stored), per-block fp64 partial sum / sum of squares
__global__ void __launch_bounds__(kAdvBlock)
adv_partial_kernel(const float* __restrict__ ret, const float* __restrict__ val, int64_t n, float* __restrict__ adv,
                   double* __restrict__ part) {
  double s = 0.0, q = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float a = ret[i] - val[i];
    adv[i] = a;
    s += (double)a;
    q += (double)a * (double)a;
  }
  __shared__ double sh_s[kAdvBlock / 32], sh_q[kAdvBlock / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
  if ((threadIdx.x & 31) == 0) { sh_s[threadIdx.x >> 5] = s; sh_q[threadIdx.x >> 5] = q; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double ts = 0.0, tq = 0.0;
    for (int w = 0; w < kAdvBlock / 32; ++w) { ts += sh_s[w]; tq += sh_q[w]; }
    part[2 * blockIdx.x] = ts;
    part[2 * blockIdx.x + 1] = tq;
  }
}

// pass 2: every block folds the partials (fixed order -> deterministic), then normalises its slice
__global__ void __launch_bounds__(kAdvBlock)
adv_apply_kernel(float* __restrict__ adv, int64_t n, const double* __restrict__ part, int nparts) {
  __shared__ float s_mean, s_inv;
  if (threadIdx.x == 0) {
    double ts = 0.0, tq = 0.0;
    for (int p = 0; p < nparts; ++p) { ts += part[2 * p]; tq += part[2 * p + 1]; }
    const double mean = ts / (double)n;
    double var = (tq - ts * mean) / (double)(n - 1);      // unbiased, as torch.Tensor.std()
    if (var < 0.0) var = 0.0;
    s_mean = (float)mean;
    s_inv = (float)sqrt(var) + 1e-8f;
  }
  __syncthreads();
  const float mean = s_mean, den = s_inv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    adv[i] = (adv[i] - mean) / den;
}

static inline int adv_grid(int64_t n) {
  int64_t g = (n + kAdvBlock * 4 - 1) / (kAdvBlock * 4);
  if (g < 1) g = 1;
  if (g > 132 * 2) g = 132 * 2;
  return (int)g;
}

}  // namespace phc

extern "C" int phc_gae(const float* fdones, const float* values, const float* rewards, const float* next_values,
                       int32_t T, int64_t N, float gamma, float tau, float* advs, float* returns, void* stream) {
  if (!fdones || !values || !rewards || !next_values || T < 0 || N < 0 || (!advs && !returns)) {
    phc_set_error("phc_gae: bad arguments"); return PHC_ERR_INVALID_ARG;
  }
  if (T == 0 || N == 0) return PHC_OK;
  const int64_t grid = (N + 31) / 32;
  phc::gae_kernel<<<(unsigned)grid, 1024, 0, static_cast<cudaStream_t>(stream)>>>(fdones, values, rewards, next_values, T, N,
                                                                                   gamma, tau, advs, returns); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "gae_kernel launch");
}

extern "C" int64_t phc_adv_norm_workspace_bytes(int64_t n) { return (int64_t)phc::adv_grid(n) * 2 * sizeof(double); }

extern "C" int phc_adv_norm(const float* returns, const float* values, int64_t n, int32_t normalize, float* advs,
                            void* workspace, void* stream) {
  if (!returns || !values || !advs || !workspace || n < 0) { phc_set_error("phc_adv_norm: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  if (normalize && n < 2) { phc_set_error("phc_adv_norm: unbiased std needs n >= 2"); return PHC_ERR_INVALID_ARG; }
  const int g = phc::adv_grid(n);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  phc::adv_partial_kernel<<<g, phc::kAdvBlock, 0, st>>>(returns, values, n, advs, static_cast<double*>(workspace)); phc_count_launches(1);
  if (normalize) phc::adv_apply_kernel<<<g, phc::kAdvBlock, 0, st>>>(advs, n, static_cast<const double*>(workspace), g); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "adv_norm kernels launch");
}
