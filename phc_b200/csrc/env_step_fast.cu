// Fused env step, steady state of the shipped SMPL configuration, with the phases ordered by INPUT ARRIVAL.
//
// What the per-warp timeline of env_step_kernel<1, 24, false, true> showed (tools/timeline_env.py):
// at 4096 envs the launch is one wave; every warp asks for its simulator block, its cached reference pose and its dof rows at
// t = 0 (13.7 MB in flight), its few scalars queue behind them, and -- a warp issues in order -- nothing computed until the first
// USE of those scalars (the frame bracket, in front of everything else) was satisfied, 2-5 us after entry.  This kernel is the same
// source expressions (env_step_shared.cuh, phc_math.cuh: operation for operation, the same warp reductions; bit-identical to the
// FAST instantiation in the -ffp-contract=off CPU emulation, to rounding on the device where nvcc contracts per kernel) in an order
// in which each phase needs only what was asked for first:
//   phase 1a [simulator block]            heading frame, SELF observation                          (humanoid.py:1994-2050)
//            -- first use of the scalar loads: frame bracket, the bracket's copies are issued; dof rows staged --
//   phase 1b [+ dof rows]                 AMP observation of the simulated character                (humanoid_amp.py:980-1060)
//   phase 2  [+ cached reference pose]    tracking errors, termination vote, reward / reset        (humanoid_im.py:1523-1608)
//   phase 3  [+ observation bracket]      blend, pose-cache row for the next step, TASK observation (humanoid_im.py:1308-1358)
// with one mbarrier per input, the simulator block requested before anything else, and the rows leaving as soon as they are
// complete (AMP slot + the first 356 floats of the observation row after phase 1).  The observation row is staged in two pieces
// because its head must not overwrite inputs that are still unread: floats [0, 356) in their own region, floats [356, 936) over
// the consumed [simulator block | cached pose] (356 * 4 bytes is the last 16-byte boundary below the self / task seam at 358).
// One warp per env, lane = body, 4 warps per CTA, 7 CTAs per SM (28 envs per SM).  On an H100: 7 x 128 threads x 64
// registers = 57 344 of 65 536, 7 x (31 168 B of shared memory at amp_dim 196 + 1 KB reserved) = 225 344 of 233 472 B, so an eighth CTA
// does not fit; 132 SMs hold 3 696 envs, and 4096 envs are one full wave plus a 400-env tail on 15 SMs (its cost is not measured
// separately: it is inside the kernel time bench.py reports).
// A/B knobs (compile-time, off by default): PHC_EXP_CACHE_LATE requests
// the cached pose together with the bracket, PHC_EXP_SCALARS_FIRST puts the scalar requests ahead of the simulator block.
// Launch conditions: exactly those of the FAST instantiation (phc_env_step checks them); reference functions replaced: as
// env_step.cu (include/phc_b200.h, PhcStepArgs).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/phc_b200.h"
#include "phc_common.cuh"
#include "phc_math.cuh"
#include "env_step_shared.cuh"

namespace phc {
namespace fast {

constexpr int kJ = 24;
constexpr int kWarps = 4;
constexpr int kCtasPerSm = 7;
constexpr int kBS = 312;                      // body_stride = round4(13 * 24)
constexpr int kD = 69;                        // 3 * (J - 1) dofs
constexpr int kSelfDim = 1 + 15 * kJ - 3;     // 358
constexpr int kObsDim = kSelfDim + 24 * kJ;   // 934
constexpr int kObsPad = 936;
constexpr int kHead = 356;                    // floats of the observation row staged in their own region
// per-env shared-memory region (floats)
constexpr int kOffState = 0;                  // simulator block                      | floats [356, 936) of the observation row are
constexpr int kOffCache = kBS;                // cached reference pose (reward time)  | staged over these two once they are consumed
constexpr int kOffOslots = 2 * kBS;           // observation bracket: 2 frame slots; slot 0 becomes the pose-cache row
constexpr int kOffDof = 4 * kBS;              // (pos, vel) pairs: 138 -> 140 floats
constexpr int kOffHead = kOffDof + 140;       // floats [0, 356) of the observation row
constexpr int kOffAmp = kOffHead + kHead;     // AMP vector (round4(amp_dim) floats), then 3 mbarriers + 2 spill floats (8 floats)

__host__ __device__ inline int env_stride(int amp_dim) { return kOffAmp + round4(amp_dim) + 8; }

__global__ void __launch_bounds__(kWarps * 32, kCtasPerSm)
env_step_fast_kernel(const __grid_constant__ PhcStepArgs a, const int amp_dim, const int stride) {
  extern __shared__ __align__(128) float smem[];
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // warp-uniform by construction
  const int env = blockIdx.x * kWarps + warp;
  if (env >= a.num_envs) return;                         // whole warp exits together; no block-level barrier is used
  float* const w_base = smem + (size_t)warp * stride;
  float* const s_state = w_base + kOffState;
  float* const s_cache = w_base + kOffCache;
  float* const s_oslots = w_base + kOffOslots;
  float* const s_dof = w_base + kOffDof;
  float* const s_head = w_base + kOffHead;
  float* const s_tail = w_base;                          // row floats [356, 936)
  float* const s_amp = w_base + kOffAmp;
  uint64_t* const bar_s = reinterpret_cast<uint64_t*>(s_amp + round4(amp_dim));
  uint64_t* const bar_c = bar_s + 1;
  uint64_t* const bar_o = bar_s + 2;
  float* const s_spill = reinterpret_cast<float*>(bar_s + 3);
  constexpr uint32_t kBlockBytes = kBS * 4u;

  if (lane == 0) {
    mbar_init(bar_s, 1);
    mbar_init(bar_c, 1);
    mbar_init(bar_o, 1);
    mbar_init_fence();
  }
  grid_dependency_wait();          // PDL: nothing above touches global memory (see env_step.cu)
  PHC_TL(0);
#ifdef PHC_EXP_TIMELINE
  if (lane == 0 && g_timeline) g_timeline[(size_t)env * 8 + 7] = smid();
#endif

  // ---- requests in the order the phases need them: simulator block, scalars, [cached pose], dof rows ----------------------------
#ifndef PHC_EXP_SCALARS_FIRST
  if (lane == 0) {
    mbar_arrive_expect_tx(bar_s, kBlockBytes);
    bulk_g2s(s_state, a.body_state + (size_t)env * a.bodies_per_env * kBodyRec, kBlockBytes, bar_s);
  }
  __syncwarp();
#endif
  const int64_t progress = a.progress[env];
  const float t_start = a.start_times[env], t_off = a.start_offsets[env];
  const V3 goff = v3(a.global_offset[3 * env + 0], a.global_offset[3 * env + 1], a.global_offset[3 * env + 2]);
  const int4 em = *reinterpret_cast<const int4*>(a.env_motion + env);
  const float m_len = __int_as_float(em.x), m_dt = __int_as_float(em.y);
  const int m_nf = em.z;
  const int64_t m_start = em.w;
#ifdef PHC_EXP_SCALARS_FIRST
  if (lane == 0) {
    mbar_arrive_expect_tx(bar_s, kBlockBytes);
    bulk_g2s(s_state, a.body_state + (size_t)env * a.bodies_per_env * kBodyRec, kBlockBytes, bar_s);
  }
  __syncwarp();
#endif
#ifndef PHC_EXP_CACHE_LATE
  if (lane == 0) {
    mbar_arrive_expect_tx(bar_c, kBlockBytes);
    bulk_g2s(s_cache, a.ref_cache + (size_t)env * kBS, kBlockBytes, bar_c);
  }
  __syncwarp();
#endif
  const float2* g_dof = reinterpret_cast<const float2*>(a.dof_state) + (size_t)env * kD;
  const float* g_force = a.dof_force + (size_t)env * kD;
  float2 dof_pv[3];
  float dof_f[3];
#pragma unroll
  for (int u = 0; u < 3; ++u) {
    const int d = lane + 32 * u;
    dof_pv[u] = (d < kD) ? g_dof[d] : make_float2(0.f, 0.f);
    dof_f[u] = (d < kD) ? g_force[d] : 0.f;
  }

  __syncwarp();
  mbar_wait(bar_s, 0);
  PHC_TL(2);

  // ================= phase 1: the simulator block alone -> self observation (1a), AMP observation (1b, + dof rows) ==============
  const bool has_body = lane < kJ;
  const int j = has_body ? lane : 0;
  const BodyRec sim = load_body(s_state + j * kBodyRec);   // stride-13 words: bank-conflict free
  const V3 root_p = v3(s_state[0], s_state[1], s_state[2]);
  const Q4 root_q = q4(s_state[3], s_state[4], s_state[5], s_state[6]);
  const float heading = heading_angle(root_q);
  const Q4 hq = quat_about_z(heading);
  const Q4 hinv = q4(0.0f, 0.0f, -hq.z, hq.w);     // quat_about_z(-heading): sin is odd, cos even -> the exact conjugate
  if (lane == 0) { s_head[0] = root_p.z; s_amp[0] = root_p.z; }
  if (has_body) {
    // self observation (compute_humanoid_observations_smpl_max); row floats 356 and 357 (body 23's last two) wait in s_spill
    float* o_pos = s_head + 1;
    float* o_rot = o_pos + 3 * (kJ - 1);
    float* o_vel = o_rot + 6 * kJ;
    float* o_ang = o_vel + 3 * kJ;
    if (j > 0) st3(o_pos + 3 * (j - 1), qrot_z(hinv, sim.p - root_p));
    const TanNorm tnm = tan_norm(qmul_zl(hinv, sim.q));
    const V3 lv = qrot_z(hinv, sim.v), lw = qrot_z(hinv, sim.w);
    st6(o_rot + 6 * j, tnm);
    st3(o_vel + 3 * j, lv);
    if (j < kJ - 1) st3(o_ang + 3 * j, lw);
    else { o_ang[3 * j] = lw.x; s_spill[0] = lw.y; s_spill[1] = lw.z; }
    if (j == 0) {                                  // AMP root columns = the root's self-observation entries (upright start)
      float* o = s_amp + 1;
      st6(o, tnm); st3(o + 6, lv); st3(o + 9, lw);
    }
  }
  __syncwarp();
  // ---- first use of the scalar / dof loads: they were requested behind the simulator block and have had phase 1a to arrive ----
  // observation bracket at the NEXT motion time (humanoid_im.py:744-752); the reward pose of this step is the cached one
  const float tn = PHC_ADD(PHC_ADD(PHC_MUL((float)(progress + 1), a.dt), t_start), t_off);
  const Bracket32 bo = frame_bracket32(tn, m_len, m_nf, m_dt);
  const float bl_o = bo.blend;
  const bool two = bo.i1 != bo.i0;                         // the last frame of a clip brackets itself: one copy, both slots alias
  const float* const po0 = s_oslots;
  const float* const po1 = two ? s_oslots + kBS : s_oslots;
  if (lane == 0) {
#ifdef PHC_EXP_CACHE_LATE
    mbar_arrive_expect_tx(bar_c, kBlockBytes);
    bulk_g2s(s_cache, a.ref_cache + (size_t)env * kBS, kBlockBytes, bar_c);
#endif
    mbar_arrive_expect_tx(bar_o, two ? 2u * kBlockBytes : kBlockBytes);
    bulk_g2s(s_oslots, a.lib.frames_body + (size_t)(m_start + bo.i0) * kBS, kBlockBytes, bar_o);
    if (two) bulk_g2s(s_oslots + kBS, a.lib.frames_body + (size_t)(m_start + bo.i1) * kBS, kBlockBytes, bar_o);
  }
  PHC_TL(1);
  float power = 0.0f;
#pragma unroll
  for (int u = 0; u < 3; ++u) {
    const int d = lane + 32 * u;
    if (d < kD) {
      s_dof[2 * d] = dof_pv[u].x;
      s_dof[2 * d + 1] = dof_pv[u].y;
      power += fabsf(dof_f[u] * dof_pv[u].y);
    }
  }
  __syncwarp();
  {
    // AMP observation of the simulated character (build_amp_observations_smpl) -> its own staging row
    const int nj = a.num_amp_joints, nk = a.num_key_bodies;
    float* o = s_amp + 1;
    if (lane < nj) {                               // nj <= 23: one joint per lane
      const int jid = a.amp_joints[lane];
      const float* dj = s_dof + 6 * jid;           // (pos, vel) pairs of the joint's 3 dofs
      st6(o + 12 + 6 * lane, tan_norm(exp_map_to_quat(v3(dj[0], dj[2], dj[4]))));
      st3(o + 12 + 6 * nj + 3 * lane, v3(dj[1], dj[3], dj[5]));
    }
    if (lane < nk) {
      const float* kb = s_state + a.key_bodies[lane] * kBodyRec;
      st3(o + 12 + 9 * nj + 3 * lane, qrot_z(hinv, v3(kb[0], kb[1], kb[2]) - root_p));
    }
  }
  float* const g_obs = a.obs + (size_t)env * a.obs_stride;
  fence_async_smem();
  __syncwarp();
  if (lane == 0) {                 // the AMP ring slot and the head of the observation row are complete: they leave now
    bulk_s2g(a.amp_out + (size_t)env * a.amp_out_stride + (a.ring_head ? (size_t)(*a.ring_head) * (size_t)amp_dim : (size_t)0), s_amp,
             (uint32_t)amp_dim * 4u);
    bulk_s2g(g_obs, s_head, (uint32_t)kHead * 4u);
    bulk_commit();
  }
  mbar_wait(bar_c, 0);
  PHC_TL(3);

  // ================= phase 2: + the cached reference pose -> reward, reset / terminate ===========================================
  {
    float e_pos = 0.f, e_rot = 0.f, e_vel = 0.f, e_ang = 0.f, dist = 0.f;
    if (has_body) {
      const BodyRec ref = load_body(s_cache + j * kBodyRec);
      const V3 dp = ref.p - sim.p;
      const float sp = dp.x * dp.x + dp.y * dp.y + dp.z * dp.z;
      e_pos = sp / 3.0f;
      const float ang = quat_angle(qmul(ref.q, qconj(sim.q)));
      e_rot = ang * ang;
      const V3 dv = ref.v - sim.v, dw = ref.w - sim.w;
      e_vel = (dv.x * dv.x + dv.y * dv.y + dv.z * dv.z) / 3.0f;
      e_ang = (dw.x * dw.x + dw.y * dw.y + dw.z * dw.z) / 3.0f;
      dist = sqrtf(sp);
    }
    const float thr = has_body ? a.term_thresh[j] : INFINITY;
    const bool fallen = __any_sync(0xffffffffu, has_body && dist > thr);
    // the four error sums in one 6-shuffle reduction: lanes 8k..8k+7 end up with sum k, finish "their" reward term
    // exp(-k * mean) (one expf sequence for the warp instead of four on lane 0) and hand it to lane 0
    const float e4 = warp_sum4(e_pos, e_rot, e_vel, e_ang, lane);
    const int sel = lane >> 3;
    const float kc = sel == 0 ? a.k_pos : (sel == 1 ? a.k_rot : (sel == 2 ? a.k_vel : a.k_ang_vel));
    const float r_mine = expf(-kc * (e4 / (float)kJ));
    const float r_pos = __shfl_sync(0xffffffffu, r_mine, 0), r_rot = __shfl_sync(0xffffffffu, r_mine, 8);
    const float r_vel = __shfl_sync(0xffffffffu, r_mine, 16), r_ang = __shfl_sync(0xffffffffu, r_mine, 24);
    power = warp_sum(power);
    if (lane == 0) {
      float rew = a.w_pos * r_pos + a.w_rot * r_rot + a.w_vel * r_vel + a.w_ang_vel * r_ang;
      float* raw = a.reward_raw + (size_t)env * 5;
      raw[0] = r_pos; raw[1] = r_rot; raw[2] = r_vel; raw[3] = r_ang;
      float pr = -a.power_coef * power;
      if (progress <= 3) pr = 0.0f;
      rew = rew + pr;
      raw[4] = pr;
      a.rew[env] = rew;
      // compute_humanoid_im_reset + the is_recovery override
      const float t_now = PHC_ADD(PHC_ADD(PHC_MUL((float)progress, a.dt), t_start), t_off);
      const bool pass_time = t_now >= m_len;
      int64_t terminated = (fallen && (progress > 1)) ? 1 : 0;
      int64_t reset = pass_time ? 1 : terminated;
      if (a.cycle_counter && !pass_time && a.cycle_counter[env] > 0) { reset = 0; terminated = 0; }
      a.reset[env] = reset;
      a.terminate[env] = terminated;
    }
  }
  __syncwarp();                    // simulator block and cached pose consumed by every lane: the row's tail may overwrite them
  if (lane == kJ - 1) { s_tail[0] = s_spill[0]; s_tail[1] = s_spill[1]; }
  mbar_wait(bar_o, 0);
  PHC_TL(4);

  // ================= phase 3: + the observation bracket -> pose cache of the next step, task observation v6 =====================
  if (has_body) {
    const BodyRec ref = blend_body(po0 + j * kBodyRec, po1 + j * kBodyRec, bl_o, goff);
    // lane j has consumed records j of both frames: slot 0 of the bracket becomes the row of the pose cache
    float* c = s_oslots + j * kBodyRec;
    st3(c, ref.p); c[3] = ref.q.x; c[4] = ref.q.y; c[5] = ref.q.z; c[6] = ref.q.w; st3(c + 7, ref.v); st3(c + 10, ref.w);
    float* tb = s_tail + (kSelfDim - kHead);
    st3(tb + 3 * j, qrot_z(hinv, ref.p - sim.p));
    st6(tb + 3 * kJ + 6 * j, tan_norm(qmul_zr(qmul_zl(hinv, qmul(ref.q, qconj(sim.q))), hq)));
    st3(tb + 9 * kJ + 3 * j, qrot_z(hinv, ref.v - sim.v));
    st3(tb + 12 * kJ + 3 * j, qrot_z(hinv, ref.w - sim.w));
    st3(tb + 15 * kJ + 3 * j, qrot_z(hinv, ref.p - root_p));
    st6(tb + 18 * kJ + 6 * j, tan_norm(qmul_zl(hinv, ref.q)));
  }
  if (lane < kObsPad - kObsDim) s_tail[kObsDim - kHead + lane] = 0.f;      // the row's pad columns are written as zeros
  fence_async_smem();
  __syncwarp();
  PHC_TL(5);
  if (lane == 0) {
    bulk_s2g(g_obs + kHead, s_tail, (uint32_t)(kObsPad - kHead) * 4u);
    bulk_s2g(a.ref_cache + (size_t)env * kBS, s_oslots, kBlockBytes);
    bulk_commit();
    bulk_wait_read0();             // the shared-memory rows must outlive the bulk reads (both groups)
  }
  PHC_TL(6);
}

}  // namespace fast
}  // namespace phc

// ------------------------------------------------------------------------------------------------------------
// launch (called by phc_env_step in env_step.cu once it has checked that the launch is the shipped steady state)
// ------------------------------------------------------------------------------------------------------------
extern "C" int phc_check_cuda(cudaError_t e, const char* what);
extern "C" void phc_count_launches(int n);

extern "C" int phc_env_step_fast_launch(const PhcStepArgs* a, int amp_dim, int pdl, void* stream) {
  using namespace phc::fast;
  const int stride = env_stride(amp_dim);
  const size_t smem = (size_t)kWarps * stride * sizeof(float);
  static size_t smem_limit = 48 * 1024;
  if (smem > smem_limit) {
    cudaError_t e = cudaFuncSetAttribute(env_step_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return phc_check_cuda(e, "cudaFuncSetAttribute(env_step_fast_kernel)");
    smem_limit = smem;
  }
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3((unsigned)((a->num_envs + kWarps - 1) / kWarps));
  lc.blockDim = dim3(kWarps * 32);
  lc.dynamicSmemBytes = smem;
  lc.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute la[1];
  la[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  la[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = la;
  lc.numAttrs = pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&lc, env_step_fast_kernel, *a, amp_dim, stride);
  if (e != cudaSuccess) return phc_check_cuda(e, "cudaLaunchKernelEx(env_step_fast_kernel)");
  phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "env_step_fast_kernel launch");
}

#ifdef PHC_EXP_TIMELINE
extern "C" PHC_API int phc_exp_set_timeline_fast(void* buf) {
  unsigned long long* p = static_cast<unsigned long long*>(buf);
  return phc_check_cuda(cudaMemcpyToSymbol(phc::g_timeline, &p, sizeof(p)), "phc_exp_set_timeline_fast");
}
#endif
