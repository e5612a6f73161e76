// Get-up schedule of HumanoidImGetup (phc/env/tasks/humanoid_im_getup.py) on the device: the reset selection of _reset_actors
// (:135-182) -- recovery episodes, fall-state starts from the pre-generated bank, reference-state starts for the rest -- and the AMP
// history of the fall starts (_init_amp_obs_default, humanoid_amp.py:570-573).  The selection is one single-CTA launch: it needs two
// ordered ranks (the k-th fall env in env order takes the k-th free state in permutation order), which one CTA computes with
// chunked ballot scans and no host round trip.  The state copies of the fall envs are a second, env-parallel launch.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/phc_b200.h"

namespace phc {
namespace getup {

constexpr int kThreads = 1024;             // the selection CTA: 32 warps
constexpr int kCopyWarps = 4;              // warps (= envs) per CTA of the state copy

// exclusive rank of `f` (0/1) among the kThreads flags of this chunk, and the chunk's total; every thread of the CTA must call it
__device__ __forceinline__ int chunk_rank(bool f, int* s_warp, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu, f);
  if (lane == 0) s_warp[warp] = __popc(b);
  __syncthreads();
  if (warp == 0) {                         // exclusive scan of the 32 warp counts
    const int v = s_warp[lane];
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    s_warp[lane] = x - v;
    if (lane == 31) s_warp[32] = x;
  }
  __syncthreads();
  const int r = s_warp[warp] + __popc(b & ((1u << lane) - 1u));
  total = s_warp[32];
  __syncthreads();                         // s_warp is reused by the next chunk
  return r;
}

// fall[e] is 1 (fall start) or 2 (recovery) while the kernel runs and ends as 0/1; ref_init doubles as the rank -> state table of
// phase 3 before it receives its own values (phase 5).  Env e is handled by the same thread in every phase.
__global__ void __launch_bounds__(kThreads)
select_kernel(const int64_t* mask, const int64_t* terminate_in, const float* u_rec, const float* u_fall, const int64_t* perm,
              const float* p_rec_dev, const float* p_fall_dev, int32_t recovery_steps, int64_t P, int64_t* available, int64_t* assignment,
              int32_t* counter, int64_t n, int64_t* progress, int64_t* reset, int64_t* terminate, int64_t* ref_init, int64_t* fall) {
  __shared__ int s_warp[33];
  const float p_rec = *p_rec_dev, p_fall = *p_fall_dev;
  // 1. free the states the resetting envs were assigned (:136; never cleared, so a stale assignment frees another env's state)
  for (int64_t e = threadIdx.x; e < n; e += kThreads)
    if (mask[e]) {
      const int64_t s = assignment[e];
      if (s >= 0 && s < P) available[s] = 0;
    }
  __syncthreads();
  // 2. recovery envs (:138-146), then fall envs among the rest (:149-154); rank of each fall env in env order
  int64_t nfall = 0;
  for (int64_t base = 0; base < n; base += kThreads) {
    const int64_t e = base + threadIdx.x;
    const bool in = e < n && mask[e] != 0;
    const bool rec = in && terminate_in[e] == 1 && u_rec[e] < p_rec;
    const bool fl = in && !rec && u_fall[e] < p_fall;
    int tot;
    const int r = chunk_rank(fl, s_warp, tot);
    if (e < n) {
      fall[e] = fl ? 1 : (rec ? 2 : 0);
      if (fl) assignment[e] = nfall + r;
    }
    nfall += tot;
  }
  // 3. the k-th free state in permutation order, k < nfall (:171-173)
  int64_t nfree = 0;
  for (int64_t base = 0; base < P && nfree < nfall; base += kThreads) {
    const int64_t i = base + threadIdx.x;
    const int64_t s = i < P ? perm[i] : 0;
    const bool fr = i < P && s >= 0 && s < P && available[s] == 0;
    int tot;
    const int r = chunk_rank(fr, s_warp, tot);
    if (fr && nfree + r < nfall) ref_init[nfree + r] = s;
    nfree += tot;
  }
  __syncthreads();
  // 4. fall envs take their state (:174-181)
  for (int64_t e = threadIdx.x; e < n; e += kThreads)
    if (fall[e] == 1) {
      // with P == N there are always enough free states (every live mark belongs to a distinct env that has not reset this time); the
      // reference asserts it (:172).  Should the bank ever run short, the env falls back to the reference-state init
      if (assignment[e] < nfree) assignment[e] = ref_init[assignment[e]];
      else { assignment[e] = 0; fall[e] = 0; }
    }
  __syncthreads();
  // 5. marks, counters, the two masks; progress / reset / terminate of fall and recovery envs (_reset_env_tensors, humanoid.py:615-617)
  for (int64_t e = threadIdx.x; e < n; e += kThreads) {
    const int64_t k = fall[e];
    const bool in = mask[e] != 0;
    if (k == 1) available[assignment[e]] = 1;
    if (k != 0) { counter[e] = recovery_steps; progress[e] = 0; reset[e] = 0; terminate[e] = 0; }
    else if (in) counter[e] = 0;                       // reference-state init (:157-160)
    ref_init[e] = (in && k == 0) ? 1 : 0;
    fall[e] = k == 1 ? 1 : 0;
  }
}

// fall envs: root record and dof state from the bank, dof velocities 0 (:174-176); one warp per env
__global__ void __launch_bounds__(kCopyWarps * 32)
copy_kernel(const int64_t* fall, const int64_t* assignment, const float* fall_root, const float* fall_dof_pos, int64_t n, float* body_state,
            int32_t bodies_per_env, float* dof_state, int32_t D) {
  const int lane = threadIdx.x & 31;
  const int64_t e = (int64_t)blockIdx.x * kCopyWarps + (threadIdx.x >> 5);
  if (e >= n || fall[e] == 0) return;
  const int64_t s = assignment[e];
  if (lane < 13) body_state[(size_t)e * bodies_per_env * 13 + lane] = fall_root[(size_t)s * 13 + lane];
  float2* d = reinterpret_cast<float2*>(dof_state) + (size_t)e * D;
  for (int i = lane; i < D; i += 32) d[i] = make_float2(fall_dof_pos[(size_t)s * D + i], 0.0f);
}

// every slot of a masked env's ring row = slot *head; one warp per env
__global__ void __launch_bounds__(kCopyWarps * 32)
ring_fill_kernel(float* ring, int64_t stride, int64_t n, int32_t S, int32_t A, const int32_t* head_dev, const int64_t* mask) {
  const int lane = threadIdx.x & 31;
  const int64_t e = (int64_t)blockIdx.x * kCopyWarps + (threadIdx.x >> 5);
  if (e >= n || mask[e] == 0) return;
  const int h = head_dev ? *head_dev : 0;
  float* row = ring + (size_t)e * stride;
  for (int i = lane; i < A; i += 32) {
    const float v = row[(size_t)h * A + i];
    for (int s = 0; s < S; ++s)
      if (s != h) row[(size_t)s * A + i] = v;
  }
}

}  // namespace getup
}  // namespace phc

extern "C" void phc_set_error(const char* msg);
extern "C" int phc_check_cuda(cudaError_t e, const char* what);
extern "C" void phc_count_launches(int n);

extern "C" int phc_getup_reset(const int64_t* mask, const int64_t* terminate_in, const float* u_rec, const float* u_fall, const int64_t* perm,
                               const float* p_rec, const float* p_fall, int32_t recovery_steps, const float* fall_root,
                               const float* fall_dof_pos, int64_t num_states, int64_t* available, int64_t* assignment,
                               int32_t* recovery_counter, int64_t n, float* body_state, int32_t bodies_per_env, float* dof_state, int32_t num_dofs,
                               int64_t* progress, int64_t* reset, int64_t* terminate, int64_t* ref_init, int64_t* fall, void* stream) {
  using namespace phc::getup;
  if (n < 0) { phc_set_error("phc_getup_reset: n < 0"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  if (!mask || !terminate_in || !u_rec || !u_fall || !perm || !p_rec || !p_fall || !fall_root || !fall_dof_pos || !available || !assignment ||
      !recovery_counter || !body_state || !dof_state || !progress || !reset || !terminate || !ref_init || !fall) {
    phc_set_error("phc_getup_reset: a required pointer is NULL"); return PHC_ERR_INVALID_ARG;
  }
  if (num_states != n) {
    phc_set_error("phc_getup_reset: the fall-state bank must hold exactly one state per env (num_states == n)"); return PHC_ERR_INVALID_ARG;
  }
  if (bodies_per_env < 1 || num_dofs < 1 || recovery_steps < 0) { phc_set_error("phc_getup_reset: bad sizes"); return PHC_ERR_INVALID_ARG; }
  if (reinterpret_cast<uintptr_t>(dof_state) & 7) { phc_set_error("phc_getup_reset: dof_state must be 8-byte aligned"); return PHC_ERR_INVALID_ARG; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  select_kernel<<<1, kThreads, 0, st>>>(mask, terminate_in, u_rec, u_fall, perm, p_rec, p_fall, recovery_steps, num_states, available, assignment,
                                        recovery_counter, n, progress, reset, terminate, ref_init, fall);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return phc_check_cuda(e, "getup select_kernel launch");
  copy_kernel<<<(unsigned)((n + kCopyWarps - 1) / kCopyWarps), kCopyWarps * 32, 0, st>>>(fall, assignment, fall_root, fall_dof_pos, n, body_state,
                                                                                           bodies_per_env, dof_state, num_dofs);
  phc_count_launches(2);
  return phc_check_cuda(cudaGetLastError(), "getup copy_kernel launch");
}

extern "C" int phc_amp_ring_fill(float* ring, int64_t ring_stride, int64_t n, int32_t num_steps, int32_t amp_dim, const int32_t* head_dev,
                                 const int64_t* mask, void* stream) {
  using namespace phc::getup;
  if (n < 0 || num_steps < 1 || amp_dim < 1 || ring_stride < (int64_t)num_steps * amp_dim) {
    phc_set_error("phc_amp_ring_fill: bad sizes (ring_stride >= num_steps * amp_dim)"); return PHC_ERR_INVALID_ARG;
  }
  if (n == 0) return PHC_OK;
  if (!ring || !mask) { phc_set_error("phc_amp_ring_fill: a required pointer is NULL"); return PHC_ERR_INVALID_ARG; }
  ring_fill_kernel<<<(unsigned)((n + kCopyWarps - 1) / kCopyWarps), kCopyWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      ring, ring_stride, n, num_steps, amp_dim, head_dev, mask);
  phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "ring_fill_kernel launch");
}
