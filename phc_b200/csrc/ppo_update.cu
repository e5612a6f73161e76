// Learner-side element-wise / reduction kernels of the PPO + AMP update (everything between the GEMMs).
// Reference (phc/...):  utils/running_mean_std.py:56-109 (RunningMeanStd), learning/common_agent.py:512-587
// (bound / actor / critic losses), learning/amp_agent.py:554-688 (calc_gradients), :732-804 (_disc_loss),
// :864-878 (_calc_disc_rewards), :848-853 (_combine_rewards); rl_games==1.1.4 (not in the reference tree):
// ModelA2CContinuousLogStd (sigma = exp(logstd), neglogp), torch_ext.policy_kl, nn.utils.clip_grad_norm_ + Adam.
//
// All of it is HBM-bound streaming over [batch, features] arrays; gradients are written pre-scaled by their loss
// coefficient and 1/batch so that the backward GEMMs need no extra pass.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/phc_b200.h"
#include "phc_common.cuh"

extern "C" void phc_set_error(const char* msg);
extern "C" int phc_check_cuda(cudaError_t e, const char* what);
extern "C" void phc_count_launches(int n);

namespace phc {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double wsumd(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------------------
// RunningMeanStd
// ---------------------------------------------------------------------------------------------------------
// y = clamp((x - mean) / sqrt(var + eps), -5, 5)   (or the un-normalise direction)
__global__ void rms_apply_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d,
                                 const double* __restrict__ mean, const double* __restrict__ var, float eps,
                                 int unnorm, float* __restrict__ y, int64_t ldy, const int64_t* __restrict__ row_idx) {
  const int64_t total = n * d;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / d;
    const int c = (int)(i - r * d);
    const float m = (float)mean[c];
    const float s = sqrtf((float)var[c] + eps);
    const int64_t rs = row_idx ? row_idx[r] : r;
    const float v = x[rs * ldx + c];
    float o;
    if (unnorm) o = s * fminf(fmaxf(v, -5.0f), 5.0f) + m;
    else o = fminf(fmaxf((v - m) / s, -5.0f), 5.0f);
    y[r * ldy + c] = o;
  }
}

// column moments in fp64 of the block's row strip: acc[y][0:d] = sum, acc[y][d:2d] = sum of squares, y = blockIdx.y (rms_merge_kernel
// adds the row strips in order, so the moments do not depend on scheduling)
__global__ void __launch_bounds__(1024) rms_moments_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d,
                                                           double* __restrict__ acc, const int64_t* __restrict__ row_idx) {
  __shared__ double s1[32][33], s2[32][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  double a = 0.0, b = 0.0;
  if (c < d)
    for (int64_t r = (int64_t)blockIdx.y * 32 + threadIdx.y; r < n; r += 32 * (int64_t)gridDim.y) {
      const double v = (double)x[(row_idx ? row_idx[r] : r) * ldx + c];
      a += v;
      b += v * v;
    }
  s1[threadIdx.y][threadIdx.x] = a;
  s2[threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  if (threadIdx.y == 0 && c < d) {
    double ta = 0.0, tb = 0.0;
    for (int i = 0; i < 32; ++i) { ta += s1[i][threadIdx.x]; tb += s2[i][threadIdx.x]; }
    acc[(int64_t)blockIdx.y * 2 * d + c] = ta;
    acc[(int64_t)blockIdx.y * 2 * d + d + c] = tb;
  }
}

// One pass over the (gathered) rows: y = clamp((x - m) / sqrt(v + eps), +-5) with the statistics (m, v) given for the APPLY, and the
// fp64 column moments of the raw rows accumulated for the UPDATE of the live statistics -- RunningMeanStd.forward in train mode
// ("update After normalization", running_mean_std.py:99-107) and AMPAgent._preproc_obs with the frozen temp copy (amp_agent.py:535-552)
// read the rows once instead of twice.  Thread (tx, ty): column blockIdx.x * 32 + tx, rows ty, ty + 32, ... of the block's row strip;
// a warp reads 128 contiguous bytes of one row per instruction, four rows in flight per thread.
__global__ void __launch_bounds__(1024) rms_apply_moments_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d,
                                                                 const double* __restrict__ mean_a, const double* __restrict__ var_a, float eps,
                                                                 float* __restrict__ y, int64_t ldy, const int64_t* __restrict__ row_idx,
                                                                 double* __restrict__ acc) {
  __shared__ double s1[32][33], s2[32][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  double a = 0.0, b = 0.0;
  if (c < d) {
    const float m = (float)mean_a[c];
    const float sd = sqrtf((float)var_a[c] + eps);
    const int64_t stride = 32 * (int64_t)gridDim.y;
    int64_t r = (int64_t)blockIdx.y * 32 + threadIdx.y;
    for (; r + 3 * stride < n; r += 4 * stride) {
      float v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { const int64_t rr = r + u * stride; v[u] = x[(row_idx ? row_idx[rr] : rr) * ldx + c]; }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        y[(r + u * stride) * ldy + c] = fminf(fmaxf((v[u] - m) / sd, -5.0f), 5.0f);
        const double dv = (double)v[u];
        a += dv; b += dv * dv;
      }
    }
    for (; r < n; r += stride) {
      const float v = x[(row_idx ? row_idx[r] : r) * ldx + c];
      y[r * ldy + c] = fminf(fmaxf((v - m) / sd, -5.0f), 5.0f);
      const double dv = (double)v;
      a += dv; b += dv * dv;
    }
  }
  s1[threadIdx.y][threadIdx.x] = a;
  s2[threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  if (threadIdx.y == 0 && c < d) {
    double ta = 0.0, tb = 0.0;
    for (int i = 0; i < 32; ++i) { ta += s1[i][threadIdx.x]; tb += s2[i][threadIdx.x]; }
    acc[(int64_t)blockIdx.y * 2 * d + c] = ta;
    acc[(int64_t)blockIdx.y * 2 * d + d + c] = tb;
  }
}

// The same two jobs (normalise; normalise + column moments) with V-wide rows per lane: V = 4 (2) consecutive columns per thread as one
// 16 (8) byte load / store when the row pitches allow it, 4 gathered rows in flight per thread.  Block = 8 warps x 32 lanes: 32 V columns,
// rows w, w + 8, ... of the block's row strip; the fp64 partial sums of the 8 warps meet in shared memory and leave as one partial per
// column and block.  Arithmetic per element is that of rms_apply_kernel ((x - mean) / sqrt(var + eps), clamp): results are bit-identical,
// the moments differ from rms_moments_kernel only in the order of the fp64 additions (a fixed order in both).
// (The scalar kernels above: 0.7 TB/s on the gathered 4096 x 1960 AMP rows, 47 us; this one is bound by the gather.)
template <int V> struct RmsVec;
template <> struct RmsVec<4> { using T = float4; };
template <> struct RmsVec<2> { using T = float2; };

template <int V, bool MOMENTS>
__global__ void __launch_bounds__(256) rms_apply_vec_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int d,
                                                            const double* __restrict__ mean_a, const double* __restrict__ var_a, float eps,
                                                            float* __restrict__ y, int64_t ldy, const int64_t* __restrict__ row_idx,
                                                            double* __restrict__ acc, int rows_per_block) {
  using VT = typename RmsVec<V>::T;
  constexpr int CW = 32 * V;
  __shared__ double s1[MOMENTS ? 8 : 1][CW], s2[MOMENTS ? 8 : 1][CW];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c0 = blockIdx.x * CW + lane * V;
  const bool full = c0 + V <= d;                   // the whole vector is inside the row (else: element by element)
  float m[V], sd[V];
  double a[V], b[V];
#pragma unroll
  for (int e = 0; e < V; ++e) {
    const int c = c0 + e < d ? c0 + e : d - 1;
    m[e] = (float)mean_a[c];
    sd[e] = sqrtf((float)var_a[c] + eps);
    a[e] = 0.0; b[e] = 0.0;
  }
  const int64_t r_begin = (int64_t)blockIdx.y * rows_per_block;
  const int64_t r_end = r_begin + rows_per_block < n ? r_begin + rows_per_block : n;
  if (c0 < d) {
    for (int64_t r = r_begin + w; r < r_end; r += 32) {
      float v[4][V];
      int64_t src[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t rr = r + 8 * u;
        src[u] = rr < r_end ? (row_idx ? row_idx[rr] : rr) : -1;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (src[u] < 0) continue;
        const float* px = x + src[u] * ldx + c0;
        if (full) {
          const VT t = *reinterpret_cast<const VT*>(px);
          const float* tf = reinterpret_cast<const float*>(&t);
#pragma unroll
          for (int e = 0; e < V; ++e) v[u][e] = tf[e];
        } else {
#pragma unroll
          for (int e = 0; e < V; ++e) v[u][e] = c0 + e < d ? px[e] : 0.f;
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (src[u] < 0) continue;
        float o[V];
#pragma unroll
        for (int e = 0; e < V; ++e) {
          o[e] = fminf(fmaxf((v[u][e] - m[e]) / sd[e], -5.0f), 5.0f);
          if (MOMENTS && c0 + e < d) { const double dv = (double)v[u][e]; a[e] += dv; b[e] += dv * dv; }
        }
        float* py = y + (r + 8 * u) * ldy + c0;
        if (full) {
          VT t;
          float* tf = reinterpret_cast<float*>(&t);
#pragma unroll
          for (int e = 0; e < V; ++e) tf[e] = o[e];
          *reinterpret_cast<VT*>(py) = t;
        } else {
#pragma unroll
          for (int e = 0; e < V; ++e) if (c0 + e < d) py[e] = o[e];
        }
      }
    }
  }
  if (MOMENTS) {
#pragma unroll
    for (int e = 0; e < V; ++e) { s1[w][lane * V + e] = a[e]; s2[w][lane * V + e] = b[e]; }
    __syncthreads();
    if (threadIdx.x < CW) {
      const int c = blockIdx.x * CW + threadIdx.x;
      if (c < d) {
        double ta = 0.0, tb = 0.0;
        for (int i = 0; i < 8; ++i) { ta += s1[i][threadIdx.x]; tb += s2[i][threadIdx.x]; }
        acc[(int64_t)blockIdx.y * 2 * d + c] = ta;
        acc[(int64_t)blockIdx.y * 2 * d + d + c] = tb;
      }
    }
  }
}

// parallel-variance merge of the batch moments into the fp64 running stats (running_mean_std.py:56-68, :99-107)
// (batch moments = the row-strip partials acc[0 .. strips - 1] added in order)
__global__ void __launch_bounds__(1024) rms_merge_kernel(const double* __restrict__ acc, int strips, int64_t n, int d,
                                                         double* __restrict__ mean, double* __restrict__ var,
                                                         double* __restrict__ count) {
  const double cnt = *count;
  const double bc = (double)n;
  const double tot = cnt + bc;
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    double s = 0.0, q = 0.0;
    for (int y = 0; y < strips; ++y) { s += acc[(int64_t)y * 2 * d + c]; q += acc[(int64_t)y * 2 * d + d + c]; }
    const double bm = s / bc;
    double bv = (q - s * bm) / (bc - 1.0);       // unbiased, torch.var default
    if (bv < 0.0) bv = 0.0;
    const double delta = bm - mean[c];
    const double new_mean = mean[c] + delta * bc / tot;
    const double m2 = var[c] * cnt + bv * bc + delta * delta * cnt * bc / tot;
    mean[c] = new_mean;
    var[c] = m2 / tot;
  }
  __syncthreads();
  if (threadIdx.x == 0) *count = tot;
}

// ---------------------------------------------------------------------------------------------------------
// Gaussian policy head (rollout): action = mu + sigma * eps, neglogp
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) gaussian_sample_kernel(const float* __restrict__ mu, int64_t ldmu,
                                                              const float* __restrict__ logstd,
                                                              const float* __restrict__ noise, int64_t n, int A,
                                                              float* __restrict__ actions, float* __restrict__ neglogp,
                                                              float* __restrict__ mus, float* __restrict__ sigmas) {
  const int64_t r = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  float acc = 0.f, ls = 0.f;
  for (int j = lane; j < A; j += 32) {
    const float m = mu[r * ldmu + j];
    const float l = logstd[j];
    const float sg = expf(l);
    const float a = m + sg * noise[r * A + j];
    actions[r * A + j] = a;
    if (mus) mus[r * A + j] = m;
    if (sigmas) sigmas[r * A + j] = sg;
    const float z = (a - m) / sg;
    acc += z * z;
    ls += l;
  }
  acc = wsum(acc);
  ls = wsum(ls);
  if (lane == 0) neglogp[r] = 0.5f * acc + 0.5f * 1.8378770664093453f * (float)A + ls;
}

// ---------------------------------------------------------------------------------------------------------
// PPO actor loss: neglogp of the stored actions under the new mu, clipped surrogate, bound loss, KL; d(loss)/d(mu)
// stats[0] += sum a_loss, [1] += sum b_loss, [2] += #clipped, [3] += sum kl, [4] += sum entropy
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ppo_actor_grad_kernel(const float* __restrict__ mu, int64_t ldmu, const float* __restrict__ logstd,
                      const float* __restrict__ actions, const float* __restrict__ old_neglogp,
                      const float* __restrict__ adv, const float* __restrict__ old_mu,
                      const float* __restrict__ old_sigma, int64_t n, int A, float e_clip, float bound_coef,
                      float inv_batch, float* __restrict__ dmu, int64_t lddmu, float* __restrict__ stats,
                      const int64_t* __restrict__ row_idx = nullptr) {
  // row_idx (optional): the minibatch is INDEX-COMPOSED -- actions / old_neglogp / adv / old_mu / old_sigma are the epoch's dataset
  // arrays and row r of the minibatch is their row row_idx[r] (mu / dmu are in minibatch order); saves six gather passes per minibatch.
  // one warp per row, rows strided over the grid; the five batch statistics are accumulated per warp, folded per block in
  // shared memory and leave with ONE atomic per block and statistic (per-row atomics on five addresses serialise: 140 us)
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  float st[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + wib; r < n; r += warps_total) {
    const int64_t rs = row_idx ? row_idx[r] : r;          // row of the dataset arrays
    float acc = 0.f, ls = 0.f, bl = 0.f, kl = 0.f;
    for (int j = lane; j < A; j += 32) {
      const float m = mu[r * ldmu + j];
      const float l = logstd[j];
      const float sg = expf(l);
      const float z = (actions[rs * A + j] - m) / sg;
      acc += z * z;
      ls += l;
      const float hi = fmaxf(m - 1.0f, 0.f), lo = fminf(m + 1.0f, 0.f);
      bl += lo * lo + hi * hi;
      const float so = old_sigma[rs * A + j], mo = old_mu[rs * A + j];
      kl += logf(so / sg + 1e-5f) + (sg * sg + (mo - m) * (mo - m)) / (2.0f * (so * so + 1e-5f)) - 0.5f;
    }
    acc = wsum(acc); ls = wsum(ls); bl = wsum(bl); kl = wsum(kl);
    const float nlp = 0.5f * acc + 0.5f * 1.8378770664093453f * (float)A + ls;
    const float ad = adv[rs];
    const float ratio = expf(old_neglogp[rs] - nlp);
    const float s1 = -ad * ratio;
    const float s2 = -ad * fminf(fmaxf(ratio, 1.0f - e_clip), 1.0f + e_clip);
    const float a_loss = fmaxf(s1, s2);
    // d a_loss / d neglogp: the un-clipped branch carries adv*ratio, the clipped one is flat (torch.max tie -> same value)
    const float g_nlp = (s1 >= s2) ? ad * ratio : 0.f;
    for (int j = lane; j < A; j += 32) {
      const float m = mu[r * ldmu + j];
      const float sg = expf(logstd[j]);
      const float dn = -(actions[rs * A + j] - m) / (sg * sg);           // d neglogp / d mu
      const float hi = fmaxf(m - 1.0f, 0.f), lo = fminf(m + 1.0f, 0.f);
      dmu[r * lddmu + j] = inv_batch * (g_nlp * dn + bound_coef * 2.0f * (hi + lo));
    }
    st[0] += a_loss;
    st[1] += bl;
    st[2] += fabsf(ratio - 1.0f) > e_clip ? 1.0f : 0.0f;
    st[3] += kl;
    st[4] += ls + 0.5f * (1.0f + 1.8378770664093453f) * (float)A;          // Normal entropy summed over actions
  }
  __shared__ float sh[8][5];
  if (lane == 0)
    for (int k = 0; k < 5; ++k) sh[wib][k] = st[k];
  __syncthreads();
  if (threadIdx.x < 5) {
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sh[w][threadIdx.x];
    atomicAdd(stats + threadIdx.x, t);
  }
}

// critic: c_loss = (ret - v)^2 (clip_value False); dv = coef * 2 (v - ret) / batch.   stats[5] += sum c_loss
__global__ void ppo_critic_grad_kernel(const float* __restrict__ v, int64_t ldv, const float* __restrict__ ret, int64_t n,
                                       float coef, float inv_batch, float* __restrict__ dv, int64_t lddv,
                                       float* __restrict__ stats, const int64_t* __restrict__ row_idx = nullptr) {
  float loss = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float d = v[i * ldv] - ret[row_idx ? row_idx[i] : i];
    loss += d * d;
    dv[i * lddv] = coef * 2.0f * d * inv_batch;
  }
  loss = wsum(loss);
  if ((threadIdx.x & 31) == 0) atomicAdd(stats + 5, loss);
}

// discriminator prediction loss: BCE-with-logits against 0 (agent + replay rows) / 1 (demo rows), 0.5 * (neg + pos)
// dl = coef * 0.5 * dBCE/dlogit / rows.  stats[6] += sum softplus(x) agent, [7] += sum softplus(-x) demo,
// [8] += #(agent logit < 0), [9] += #(demo logit > 0)
__global__ void disc_logit_grad_kernel(const float* __restrict__ logit, int64_t ld, int64_t n_agent, int64_t n_demo,
                                       float coef, float* __restrict__ dlogit, int64_t ldd, float* __restrict__ stats) {
  float la = 0.f, lp = 0.f, ca = 0.f, cd = 0.f;
  const int64_t n = n_agent + n_demo;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float x = logit[i * ld];
    const float sp = fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)));          // softplus(x)
    const float sig = 1.0f / (1.0f + expf(-x));
    if (i < n_agent) {
      la += sp;
      ca += (x < 0.f) ? 1.f : 0.f;
      dlogit[i * ldd] = coef * 0.5f * sig / (float)n_agent;
    } else {
      lp += sp - x;                                                    // softplus(-x)
      cd += (x > 0.f) ? 1.f : 0.f;
      dlogit[i * ldd] = coef * 0.5f * (sig - 1.0f) / (float)n_demo;
    }
  }
  la = wsum(la); lp = wsum(lp); ca = wsum(ca); cd = wsum(cd);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(stats + 6, la); atomicAdd(stats + 7, lp); atomicAdd(stats + 8, ca); atomicAdd(stats + 9, cd);
  }
}

// disc reward (amp_agent.py:864-878) fused with _combine_rewards (:848-853):
//   r = w_task * task + w_disc * scale * (-log(max(1 - sigmoid(logit), 1e-4)))
__global__ void disc_reward_kernel(const float* __restrict__ logit, int64_t ld, const float* __restrict__ task, int64_t n,
                                   float scale, float w_task, float w_disc, float* __restrict__ disc_r,
                                   float* __restrict__ combined) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float prob = 1.0f / (1.0f + expf(-logit[i * ld]));
    const float dr = -logf(fmaxf(1.0f - prob, 0.0001f)) * scale;
    if (disc_r) disc_r[i] = dr;
    if (combined) combined[i] = w_task * task[i] + w_disc * dr;
  }
}

// u[b, j] = (h[b, j] > 0) ? w[j] : 0        (first step of d logit / d input through a ReLU MLP)
__global__ void relu_mask_row_kernel(const float* __restrict__ h, int64_t ldh, const float* __restrict__ w, int64_t n, int d,
                                     float* __restrict__ u, int64_t ldu) {
  const int64_t total = n * d;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / d;
    const int c = (int)(i - r * d);
    u[r * ldu + c] = h[r * ldh + c] > 0.f ? w[c] : 0.f;
  }
}

// x *= alpha in place and stats[slot] += sum(x_before^2)      (gradient penalty: g -> dP/dg, keeps sum ||g||^2)
__global__ void scale_sumsq_kernel(float* __restrict__ x, int64_t ld, int64_t n, int d, float alpha, float* __restrict__ stat) {
  const int64_t total = n * d;
  float s = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / d;
    const int c = (int)(i - r * d);
    const float v = x[r * ld + c];
    s += v * v;
    x[r * ld + c] = v * alpha;
  }
  s = wsum(s);
  if ((threadIdx.x & 31) == 0) atomicAdd(stat, s);
}

// y += alpha * x over a strided [rows, cols] block (weight decay / logit regulariser gradients)
__global__ void axpy2d_kernel(const float* __restrict__ x, int64_t ldx, float* __restrict__ y, int64_t ldy, int64_t rows,
                              int cols, float alpha, float* __restrict__ sumsq_stat) {
  const int64_t total = rows * cols;
  float s = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cols;
    const int c = (int)(i - r * cols);
    const float v = x[r * ldx + c];
    y[r * ldy + c] += alpha * v;
    s += v * v;
  }
  if (sumsq_stat) {
    s = wsum(s);
    if ((threadIdx.x & 31) == 0) atomicAdd(sumsq_stat, s);
  }
}

// ---------------------------------------------------------------------------------------------------------
// global-norm clip + Adam on the flat parameter bucket
// ---------------------------------------------------------------------------------------------------------
// sum of squares in fp64: one partial per block (warps added in order), then sum_parts_kernel adds the blocks in order -- the norm
// that scales the clip does not depend on scheduling
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ g, int64_t n, double* __restrict__ part) {
  __shared__ double w[8];
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double v = (double)g[i];
    s += v * v;
  }
  s = wsumd(s);
  if ((threadIdx.x & 31) == 0) w[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += w[i];
    part[blockIdx.x] = t;
  }
}
__global__ void sum_parts_kernel(const double* __restrict__ part, int parts, double* __restrict__ out) {
  double t = 0.0;
  for (int i = 0; i < parts; ++i) t += part[i];
  *out = t;
}

// torch.nn.utils.clip_grad_norm_(max_norm) + torch.optim.Adam(lr, betas, eps, weight_decay=0) in one pass.
// grad_scale multiplies the gradient first (1/world_size after a sum all-reduce).  sumsq is the squared norm of
// the UNSCALED g (phc_grad_sumsq).  step_count is the 1-based Adam step.
__global__ void adam_clip_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                 float* __restrict__ v, int64_t n, const double* __restrict__ sumsq, float grad_scale,
                                 float max_norm, float lr, float beta1, float beta2, float eps, float bc1, float bc2_sqrt) {
  float clip = 1.0f;
  if (max_norm > 0.f) {
    const float total = grad_scale * (float)sqrt(*sumsq);          // norm of the scaled gradient
    clip = fminf(max_norm / (total + 1e-6f), 1.0f);
  }
  const float gs = grad_scale * clip;
  const float step = lr / bc1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float gi = g[i] * gs;
    const float mi = beta1 * m[i] + (1.0f - beta1) * gi;
    const float vi = beta2 * v[i] + (1.0f - beta2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] = p[i] - step * (mi / (sqrtf(vi) / bc2_sqrt + eps));
  }
}

// HumanoidImMCP.step (phc/env/tasks/humanoid_im_mcp.py:79-82): actions[n, a] = sum_k weights[n, k] * prim[k][n, a]
// prim: K activation matrices with a common row stride, stacked `prim_stride` floats apart.
__global__ void mcp_combine_kernel(const float* __restrict__ w, int64_t ldw, const float* __restrict__ prim, int64_t ldp,
                                   int64_t prim_stride, int64_t n, int K, int A, int discrete, float* __restrict__ out, int64_t ldo) {
  const int64_t total = n * A;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / A;
    const int c = (int)(i - r * A);
    float acc = 0.f;
    if (discrete) {      // discrete_moe (humanoid_im_mcp.py:70-72): one-hot of the first arg-max weight
      int best = 0;
      float bw = w[r * ldw];
      for (int k = 1; k < K; ++k) { const float v = w[r * ldw + k]; if (v > bw) { bw = v; best = k; } }
      for (int k = 0; k < K; ++k) acc = __fadd_rn(acc, __fmul_rn(k == best ? 1.f : 0.f, prim[k * prim_stride + r * ldp + c]));
    } else {
      for (int k = 0; k < K; ++k)      // product rounded, then added: the reference's weights[:, :, None] * x_all followed by sum(dim=1)
        acc = __fadd_rn(acc, __fmul_rn(w[r * ldw + k], prim[k * prim_stride + r * ldp + c]));
    }
    out[r * ldo + c] = acc;
  }
}

// Humanoid._action_to_pd_targets (humanoid.py:1711-1713) with the surrounding pre_physics_step logic (:1540-1556):
//   pd_tar = pd_action_offset + pd_action_scale * action      (product rounded, then the sum: torch evaluates it as two ops)
// reduce_action: the policy emits only the dofs listed in action_idx, all others see action 0 (-> the offset);
// zero_mask: dofs of frozen hands / toes are forced to 0 after the affine map.
__global__ void pd_targets_kernel(const float* __restrict__ act, int64_t lda, int64_t n, int D, int A,
                                  const int32_t* __restrict__ dof_of_action, const float* __restrict__ offset,
                                  const float* __restrict__ scale, const uint8_t* __restrict__ zero_mask, float* __restrict__ out,
                                  int64_t ldo) {
  const int64_t total = n * D;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / D;
    const int d = (int)(i - r * D);
    float a;
    if (dof_of_action) {          // reduce_action: dof_of_action[d] = column of the action that drives dof d, or -1
      const int c = dof_of_action[d];
      a = c >= 0 ? act[r * lda + c] : 0.0f;
    } else {
      a = d < A ? act[r * lda + d] : 0.0f;
    }
    float t = __fadd_rn(offset[d], __fmul_rn(scale[d], a));
    if (zero_mask && zero_mask[d]) t = 0.0f;
    out[r * ldo + d] = t;
  }
}

// backward of the activation that ends the MCP composer (amp_network_mcp_builder.py:57-63, ending_act):
// ReLU: dy[r, c] = aux[r, c] > 0 ? dy[r, c] : 0 (aux = output);  SiLU: dy[r, c] *= silu'(aux[r, c]) (aux = pre-activation)
__global__ void act_backward_kernel(float* __restrict__ dy, int64_t ldd, const float* __restrict__ y, int64_t ldy, int64_t n, int d,
                                    int act) {
  const int64_t total = n * d;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / d;
    const int c = (int)(i - r * d);
    if (act == PHC_ACT_SILU) dy[r * ldd + c] *= silu_grad_f(y[r * ldy + c]);
    else if (!(y[r * ldy + c] > 0.f)) dy[r * ldd + c] = 0.f;
  }
}

constexpr int RMS_MAX_STRIPS = 32;      // row strips of the column-moment kernels: one fp64 partial pair per strip in the workspace
constexpr int SUMSQ_SLOTS = 8, SUMSQ_MAX_PARTS = 132 * 8;
__device__ double g_sumsq_parts[SUMSQ_SLOTS][SUMSQ_MAX_PARTS];

static inline int ew_grid(int64_t total, int block = 256) {
  int64_t g = (total + block - 1) / block;
  if (g > 132 * 8) g = 132 * 8;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace phc

using namespace phc;
#define ST(s) static_cast<cudaStream_t>(s)

// vector width of rms_apply_vec_kernel for these pitches / pointers (0: use the scalar kernels)
static int rms_vec_width(const float* x, int64_t ldx, const float* y, int64_t ldy) {
  const uintptr_t px = reinterpret_cast<uintptr_t>(x), py = reinterpret_cast<uintptr_t>(y);
  if (!(ldx & 3) && !(ldy & 3) && !(px & 15) && !(py & 15)) return 4;
  if (!(ldx & 1) && !(ldy & 1) && !(px & 7) && !(py & 7)) return 2;
  return 0;
}
// rows per block so that the grid is a few waves of 256-thread blocks (multiple of 32 rows: 4 rows in flight x 8 warps)
static int rms_rows_per_block(int64_t n, int col_blocks) {
  int64_t want = (int64_t)132 * 8 / (col_blocks > 0 ? col_blocks : 1);
  if (want < 1) want = 1;
  int64_t rows = (n + want - 1) / want;
  rows = (rows + 31) / 32 * 32;
  if (rows < 32) rows = 32;
  return (int)rows;
}

extern "C" int phc_rms_apply(const float* x, int64_t ldx, int64_t n, int32_t d, const double* mean, const double* var,
                             float eps, int32_t unnorm, float* y, int64_t ldy, const int64_t* row_idx, void* stream) {
  if (!x || !mean || !var || !y || n < 0 || d < 1 || ldx < d || ldy < d) { phc_set_error("phc_rms_apply: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  const int V = unnorm ? 0 : rms_vec_width(x, ldx, y, ldy);
  if (V) {
    const int cb = (d + 32 * V - 1) / (32 * V), rpb = rms_rows_per_block(n, cb);
    const dim3 grid(cb, (unsigned)((n + rpb - 1) / rpb));
    if (V == 4) rms_apply_vec_kernel<4, false><<<grid, 256, 0, ST(stream)>>>(x, ldx, n, d, mean, var, eps, y, ldy, row_idx, nullptr, rpb);
    else rms_apply_vec_kernel<2, false><<<grid, 256, 0, ST(stream)>>>(x, ldx, n, d, mean, var, eps, y, ldy, row_idx, nullptr, rpb);
    phc_count_launches(1);
    return phc_check_cuda(cudaGetLastError(), "rms_apply_vec_kernel");
  }
  rms_apply_kernel<<<ew_grid(n * d), 256, 0, ST(stream)>>>(x, ldx, n, d, mean, var, eps, unnorm, y, ldy, row_idx); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "rms_apply_kernel");
}

extern "C" int64_t phc_rms_workspace_bytes(int32_t d) { return (int64_t)RMS_MAX_STRIPS * 2 * d * sizeof(double); }

extern "C" int phc_rms_update(const float* x, int64_t ldx, int64_t n, int32_t d, double* mean, double* var, double* count,
                              void* workspace, const int64_t* row_idx, void* stream) {
  if (!x || !mean || !var || !count || !workspace || n < 2 || d < 1 || ldx < d) { phc_set_error("phc_rms_update: bad arguments (needs n >= 2)"); return PHC_ERR_INVALID_ARG; }
  double* acc = static_cast<double*>(workspace);
  int gy = (int)((n + 1023) / 1024); if (gy > RMS_MAX_STRIPS) gy = RMS_MAX_STRIPS; if (gy < 1) gy = 1;
  rms_moments_kernel<<<dim3((d + 31) / 32, gy), dim3(32, 32), 0, ST(stream)>>>(x, ldx, n, d, acc, row_idx); phc_count_launches(1);
  rms_merge_kernel<<<1, 1024, 0, ST(stream)>>>(acc, gy, n, d, mean, var, count); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "rms_update kernels");
}

extern "C" int phc_rms_apply_update(const float* x, int64_t ldx, int64_t n, int32_t d, const double* mean_apply, const double* var_apply,
                                    float eps, float* y, int64_t ldy, const int64_t* row_idx, double* mean, double* var, double* count,
                                    void* workspace, void* stream) {
  if (!x || !mean_apply || !var_apply || !y || !mean || !var || !count || !workspace || n < 2 || d < 1 || ldx < d || ldy < d) {
    phc_set_error("phc_rms_apply_update: bad arguments (needs n >= 2)"); return PHC_ERR_INVALID_ARG;
  }
  double* acc = static_cast<double*>(workspace);
  const int V = rms_vec_width(x, ldx, y, ldy);
  int gy;
  if (V) {
    const int cb = (d + 32 * V - 1) / (32 * V);
    int rpb = rms_rows_per_block(n, cb);
    if ((n + rpb - 1) / rpb > RMS_MAX_STRIPS) rpb = (int)(((n + RMS_MAX_STRIPS - 1) / RMS_MAX_STRIPS + 31) / 32 * 32);
    gy = (int)((n + rpb - 1) / rpb);
    const dim3 grid(cb, (unsigned)gy);
    if (V == 4) rms_apply_vec_kernel<4, true><<<grid, 256, 0, ST(stream)>>>(x, ldx, n, d, mean_apply, var_apply, eps, y, ldy, row_idx, acc, rpb);
    else rms_apply_vec_kernel<2, true><<<grid, 256, 0, ST(stream)>>>(x, ldx, n, d, mean_apply, var_apply, eps, y, ldy, row_idx, acc, rpb);
  } else {
    gy = (int)((n + 255) / 256); if (gy > 24) gy = 24; if (gy < 1) gy = 1;
    rms_apply_moments_kernel<<<dim3((d + 31) / 32, gy), dim3(32, 32), 0, ST(stream)>>>(x, ldx, n, d, mean_apply, var_apply, eps, y, ldy, row_idx, acc);
  }
  phc_count_launches(1);
  rms_merge_kernel<<<1, 1024, 0, ST(stream)>>>(acc, gy, n, d, mean, var, count); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "rms_apply_update kernels");
}

extern "C" int phc_gaussian_sample(const float* mu, int64_t ldmu, const float* logstd, const float* noise, int64_t n,
                                   int32_t A, float* actions, float* neglogp, float* mus, float* sigmas, void* stream) {
  if (!mu || !logstd || !noise || !actions || !neglogp || n < 0 || A < 1 || ldmu < A) { phc_set_error("phc_gaussian_sample: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  gaussian_sample_kernel<<<(unsigned)((n + 3) / 4), 128, 0, ST(stream)>>>(mu, ldmu, logstd, noise, n, A, actions, neglogp, mus, sigmas); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "gaussian_sample_kernel");
}

extern "C" int phc_ppo_actor_grad(const float* mu, int64_t ldmu, const float* logstd, const float* actions,
                                  const float* old_neglogp, const float* adv, const float* old_mu, const float* old_sigma,
                                  int64_t n, int32_t A, float e_clip, float bound_coef, float inv_batch, float* dmu,
                                  int64_t lddmu, float* stats, void* stream) {
  if (!mu || !logstd || !actions || !old_neglogp || !adv || !old_mu || !old_sigma || !dmu || !stats || n < 0 || A < 1 || ldmu < A || lddmu < A) {
    phc_set_error("phc_ppo_actor_grad: bad arguments"); return PHC_ERR_INVALID_ARG;
  }
  if (n == 0) return PHC_OK;
  ppo_actor_grad_kernel<<<(unsigned)((n + 7) / 8 < 132 * 4 ? (n + 7) / 8 : 132 * 4), 256, 0, ST(stream)>>>(mu, ldmu, logstd, actions, old_neglogp, adv, old_mu, old_sigma, n, A,
                                                                         e_clip, bound_coef, inv_batch, dmu, lddmu, stats); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "ppo_actor_grad_kernel");
}

extern "C" int phc_ppo_grads_gather(const float* mu, int64_t ldmu, const float* logstd, const float* actions, const float* old_neglogp,
                                    const float* adv, const float* old_mu, const float* old_sigma, const float* v, int64_t ldv,
                                    const float* ret, const int64_t* row_idx, int64_t n, int32_t A, float e_clip, float bound_coef,
                                    float critic_coef, float inv_batch, float* dmu, int64_t lddmu, float* dv, int64_t lddv, float* stats,
                                    void* stream) {
  if (!mu || !logstd || !actions || !old_neglogp || !adv || !old_mu || !old_sigma || !v || !ret || !row_idx || !dmu || !dv || !stats || n < 0 ||
      A < 1 || ldmu < A || lddmu < A || ldv < 1 || lddv < 1) {
    phc_set_error("phc_ppo_grads_gather: bad arguments"); return PHC_ERR_INVALID_ARG;
  }
  if (n == 0) return PHC_OK;
  ppo_actor_grad_kernel<<<(unsigned)((n + 7) / 8 < 132 * 4 ? (n + 7) / 8 : 132 * 4), 256, 0, ST(stream)>>>(mu, ldmu, logstd, actions, old_neglogp, adv, old_mu, old_sigma, n, A,
                                                                         e_clip, bound_coef, inv_batch, dmu, lddmu, stats, row_idx); phc_count_launches(1);
  ppo_critic_grad_kernel<<<ew_grid(n), 256, 0, ST(stream)>>>(v, ldv, ret, n, critic_coef, inv_batch, dv, lddv, stats, row_idx); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "ppo_grads_gather kernels");
}

extern "C" int phc_ppo_critic_grad(const float* v, int64_t ldv, const float* ret, int64_t n, float coef, float inv_batch,
                                   float* dv, int64_t lddv, float* stats, void* stream) {
  if (!v || !ret || !dv || !stats || n < 0 || ldv < 1 || lddv < 1) { phc_set_error("phc_ppo_critic_grad: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  ppo_critic_grad_kernel<<<ew_grid(n), 256, 0, ST(stream)>>>(v, ldv, ret, n, coef, inv_batch, dv, lddv, stats); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "ppo_critic_grad_kernel");
}

extern "C" int phc_disc_logit_grad(const float* logit, int64_t ld, int64_t n_agent, int64_t n_demo, float coef,
                                   float* dlogit, int64_t ldd, float* stats, void* stream) {
  if (!logit || !dlogit || !stats || n_agent < 1 || n_demo < 1 || ld < 1 || ldd < 1) { phc_set_error("phc_disc_logit_grad: bad arguments"); return PHC_ERR_INVALID_ARG; }
  disc_logit_grad_kernel<<<ew_grid(n_agent + n_demo), 256, 0, ST(stream)>>>(logit, ld, n_agent, n_demo, coef, dlogit, ldd, stats); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "disc_logit_grad_kernel");
}

extern "C" int phc_disc_reward(const float* logit, int64_t ld, const float* task_rewards, int64_t n, float scale,
                               float w_task, float w_disc, float* disc_rewards, float* combined, void* stream) {
  if (!logit || n < 0 || ld < 1 || (combined && !task_rewards) || (!disc_rewards && !combined)) { phc_set_error("phc_disc_reward: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  disc_reward_kernel<<<ew_grid(n), 256, 0, ST(stream)>>>(logit, ld, task_rewards, n, scale, w_task, w_disc, disc_rewards, combined); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "disc_reward_kernel");
}

extern "C" int phc_relu_mask_row(const float* h, int64_t ldh, const float* w, int64_t n, int32_t d, float* u, int64_t ldu,
                                 void* stream) {
  if (!h || !w || !u || n < 0 || d < 1 || ldh < d || ldu < d) { phc_set_error("phc_relu_mask_row: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  relu_mask_row_kernel<<<ew_grid(n * d), 256, 0, ST(stream)>>>(h, ldh, w, n, d, u, ldu); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "relu_mask_row_kernel");
}

extern "C" int phc_scale_sumsq(float* x, int64_t ld, int64_t n, int32_t d, float alpha, float* stat, void* stream) {
  if (!x || !stat || n < 0 || d < 1 || ld < d) { phc_set_error("phc_scale_sumsq: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  scale_sumsq_kernel<<<ew_grid(n * d), 256, 0, ST(stream)>>>(x, ld, n, d, alpha, stat); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "scale_sumsq_kernel");
}

extern "C" int phc_axpy2d(const float* x, int64_t ldx, float* y, int64_t ldy, int64_t rows, int32_t cols, float alpha,
                          float* sumsq_stat, void* stream) {
  if (!x || !y || rows < 0 || cols < 1 || ldx < cols || ldy < cols) { phc_set_error("phc_axpy2d: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (rows == 0) return PHC_OK;
  axpy2d_kernel<<<ew_grid(rows * cols), 256, 0, ST(stream)>>>(x, ldx, y, ldy, rows, cols, alpha, sumsq_stat); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "axpy2d_kernel");
}

extern "C" int phc_grad_sumsq(const float* g, int64_t n, double* out, void* stream) {
  if (!g || !out || n < 0) { phc_set_error("phc_grad_sumsq: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) { cudaMemsetAsync(out, 0, sizeof(double), ST(stream)); return PHC_OK; }
  static double* base = nullptr;
  static unsigned int launch_no = 0;
  if (!base) {
    void* p = nullptr;
    cudaError_t e = cudaGetSymbolAddress(&p, g_sumsq_parts);
    if (e != cudaSuccess) return phc_check_cuda(e, "cudaGetSymbolAddress(g_sumsq_parts)");
    base = static_cast<double*>(p);
  }
  double* part = base + (size_t)(launch_no++ % SUMSQ_SLOTS) * SUMSQ_MAX_PARTS;     // calls in flight on different streams: different slots
  const int grid = ew_grid(n);
  sumsq_kernel<<<grid, 256, 0, ST(stream)>>>(g, n, part);
  sum_parts_kernel<<<1, 1, 0, ST(stream)>>>(part, grid, out); phc_count_launches(2);
  return phc_check_cuda(cudaGetLastError(), "sumsq_kernel");
}

extern "C" int phc_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n,
                             const double* grad_sumsq, float grad_scale, float max_norm, float lr, float beta1, float beta2,
                             float eps, int64_t step, void* stream) {
  if (!params || !grads || !exp_avg || !exp_avg_sq || n < 0 || step < 1 || (max_norm > 0.f && !grad_sumsq)) {
    phc_set_error("phc_adam_step: bad arguments"); return PHC_ERR_INVALID_ARG;
  }
  if (n == 0) return PHC_OK;
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const double bc2 = 1.0 - pow((double)beta2, (double)step);
  adam_clip_kernel<<<ew_grid(n), 256, 0, ST(stream)>>>(params, grads, exp_avg, exp_avg_sq, n, grad_sumsq, grad_scale, max_norm, lr,
                                                       beta1, beta2, eps, (float)bc1, (float)sqrt(bc2)); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "adam_clip_kernel");
}

extern "C" int phc_mcp_combine(const float* weights, int64_t ldw, const float* prim, int64_t ldp, int64_t prim_stride, int64_t n,
                               int32_t K, int32_t A, int32_t discrete, float* out, int64_t ldo, void* stream) {
  if (n == 0) return PHC_OK;                       // empty batch: nothing to validate, nothing to launch
  if (!weights || !prim || !out || n < 0 || K < 1 || A < 1 || ldw < K || ldp < A || ldo < A) { phc_set_error("phc_mcp_combine: bad arguments"); return PHC_ERR_INVALID_ARG; }
  mcp_combine_kernel<<<ew_grid(n * A), 256, 0, ST(stream)>>>(weights, ldw, prim, ldp, prim_stride, n, K, A, discrete, out, ldo); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "mcp_combine_kernel");
}

extern "C" int phc_pd_targets(const float* actions, int64_t lda, int64_t n, int32_t num_dofs, int32_t num_actions,
                              const int32_t* dof_of_action, const float* offset, const float* scale, const uint8_t* zero_mask,
                              float* out, int64_t ldo, void* stream) {
  if (!actions || !offset || !scale || !out || n < 0 || num_dofs < 1 || num_actions < 1 || lda < num_actions || ldo < num_dofs ||
      (!dof_of_action && num_actions != num_dofs)) {
    phc_set_error("phc_pd_targets: bad arguments (without dof_of_action the action must have one column per dof)");
    return PHC_ERR_INVALID_ARG;
  }
  if (n == 0) return PHC_OK;
  int64_t g = (n * num_dofs + 255) / 256; if (g > 132 * 8) g = 132 * 8;
  phc::pd_targets_kernel<<<(unsigned)g, 256, 0, static_cast<cudaStream_t>(stream)>>>(actions, lda, n, num_dofs, num_actions, dof_of_action, offset, scale,
                                                                                  zero_mask, out, ldo); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "pd_targets_kernel launch");
}

extern "C" int phc_act_backward(float* dy, int64_t ldd, const float* aux, int64_t ldaux, int64_t n, int32_t d, int32_t act, void* stream) {
  if (n == 0) return PHC_OK;
  if (!dy || !aux || n < 0 || d < 1 || ldd < d || ldaux < d || (act != PHC_ACT_RELU && act != PHC_ACT_SILU)) { phc_set_error("phc_act_backward: bad arguments"); return PHC_ERR_INVALID_ARG; }
  act_backward_kernel<<<ew_grid(n * d), 256, 0, ST(stream)>>>(dy, ldd, aux, ldaux, n, d, act); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "act_backward_kernel");
}
