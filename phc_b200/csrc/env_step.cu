// Fused post-physics env step for HumanoidIm: motion-library query (2 brackets) + self obs + task obs v6 +
// tracking/power reward + reset/terminate + AMP observation (+ window shift) in ONE launch.
// Reference functions replaced: see include/phc_b200.h (PhcStepArgs).
//
// Mapping: one warp per environment, lane j = body j (J <= 32).  Per env the kernel moves, for J = 24 / T = 1:
//   reads  1248 B simulator state + <= 4 x 1248 B motion frames (3 distinct in steady state: the reward bracket
//          [k, k+1] and the obs bracket [k+1, k+2] share a frame) + 552 B dof state + 276 B dof force + ~100 B scalars
//   writes 3736 B observation + 40 B reward/reset + 784 B AMP vector (+ optional window shift / ref_* side buffers)
// -> HBM-bound (about 250 FLOP per 52-byte body).  Blocks are staged into shared memory with TMA 1-D bulk copies
// (cp.async.bulk + mbarrier: no register staging, one elected lane issues), de-interleaved from shared memory with
// stride-13 reads (conflict free), results are staged as one observation row in shared memory and leave with
// coalesced 8-byte stores.  28 envs are resident per SM at J = 24 so N = 4096 fills 147 SMs (a little over one wave on an H100's 132).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/phc_b200.h"
#include "phc_common.cuh"
#include "phc_math.cuh"
#include "env_step_shared.cuh"

namespace phc {

#ifndef PHC_EXP_WARPS            // experiment knob (phc_b200.build.build_variant): warps (= envs) per CTA
#define PHC_EXP_WARPS 4
#endif
constexpr int kWarpsPerCta = PHC_EXP_WARPS;
constexpr int kMinCtasPerSm = 28 / PHC_EXP_WARPS;   // 28 envs resident per SM: 4096 envs fill 147 SMs
struct StepLayout {      // per-warp shared-memory carve-up, in floats (all multiples of 4 -> 16-byte aligned)
  int rslots;            // 2 frame slots of the reward bracket            | the observation row (T == 1) is
  int state;             // J*13 rounded up: the env's simulator block     | staged over these two regions once
  int oslots;            // 2T frame slots of the observation bracket(s)     their contents have been consumed
  int dof;               // 2*D rounded up (pos, vel interleaved as in dof_state)
  int amp;               // A rounded up
  int obs;               // separate obs row (0 when it aliases rslots+state)
  int total;             // sum + 4 (mbarrier)
};

__host__ __device__ inline StepLayout make_layout(int J, int T, int body_stride, int A, int obs_dim, bool alias_obs, int D = 0) {
  StepLayout L;
  L.rslots = 2 * body_stride;
  L.state = round4(J * kBodyRec);
  L.oslots = 2 * T * body_stride;
  L.dof = round4(2 * (D > 0 ? D : 3 * (J - 1)));
  L.amp = round4(A > 0 ? A : 4);
  L.obs = alias_obs ? 0 : round4(obs_dim);
  L.total = L.rslots + L.state + L.oslots + L.dof + L.amp + L.obs + 4;
  return L;
}

// JT > 0: the body count is a compile-time constant (24 = SMPL, 20 = H1): record strides, segment offsets of the observation
// row and the shared-memory carve-up fold into immediates; JT == 0 is the generic runtime-J build.
// GETUP: the env_im_getup_mcp.yaml extras (PHC_FLAG_ZERO_OUT_FAR / PHC_FLAG_CYCLE_MOTION, T == 1, spherical joints).  A template
// parameter so the plain instantiations keep exactly the instruction stream they had without it.
// FAST: the steady-state launch of the shipped SMPL configuration (phc_env_step checks every condition): flags exactly
// kFastFlags, pose cache on, no env mask, per-env motion records given, every row movable as a TMA bulk copy, no ref_*
// side buffers.  All of that becomes compile-time, so the flag tests, the non-cache reward path, the row-store fallbacks and
// their predicates / branches leave the instruction stream (the arithmetic is the same code, operation for operation).
// KP: the keypoint-only task observation v7 (PHC_FLAG_TASK_OBS_KP) instead of v6; a template parameter for the same reason as GETUP.
// REC: the get-up schedule (HumanoidImGetup, humanoid_im_getup.py): PHC_FLAG_RECOVERY on a step launch (recovery counter, reset
// override, frozen progress) and PHC_FLAG_AMP_CURRENT on the observation-only launch (the AMP vector of the current state); again a
// template parameter so that every other instantiation keeps its instruction stream.
template <int T_MAX, int JT, bool GETUP = false, bool FAST = false, bool KP = false, bool REC = false>
__global__ void __launch_bounds__(kWarpsPerCta * 32, kMinCtasPerSm)
env_step_kernel(const __grid_constant__ PhcStepArgs a, const int obs_dim, const int self_dim, const int amp_dim,
                const bool alias_obs_rt, const bool state_bulk_ok_rt) {
  extern __shared__ __align__(128) float smem[];
  // the warp index through a shuffle: the compiler then KNOWS it (and the env index, and every pointer derived from it) is
  // warp-uniform, keeps them in uniform registers and issues the bulk copies straight from there instead of wrapping each
  // one in a vote + R2UR.BROADCAST loop
#ifdef PHC_EXP_NO_UNIFORM_WARP      // A/B build (phc_b200.build.build_variant): the round-1 form
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#else
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
#endif
  const int env = blockIdx.x * kWarpsPerCta + warp;
  if (env >= a.num_envs) return;                       // whole warp exits together; no block-level barrier is used
#if defined(PHC_EXP_EXIT) && PHC_EXP_EXIT == 1      // floor experiment: launch + CTA ramp only
  grid_dependency_wait();
  return;
#endif
#ifdef PHC_EXP_TIMELINE
  if (lane == 0 && g_timeline) g_timeline[(size_t)env * 8 + 7] = smid();
#endif
  if (!FAST && a.only_where) {                         // masked subset (reset path): the mask is the previous kernel's output
    grid_dependency_wait();
    if (a.only_where[env] == 0) return;
  }
  const uint32_t flags = FAST ? kFastFlags : a.flags;
  const bool alias_obs = FAST ? true : alias_obs_rt;
  const bool state_bulk_ok = FAST ? true : state_bulk_ok_rt;
  const bool obs_only = flags & PHC_FLAG_OBS_ONLY;

  // JT > 0 is the SMPL specialisation (spherical joints, no extend bodies); robots (hinge joints, E extend bodies that enter
  // the tracking reward as lanes J..J+E-1) take the run-time build
  const int J = JT > 0 ? JT : a.lib.num_bodies;
  const int E = JT > 0 ? 0 : a.lib.num_ext_bodies;
  const bool robot = JT > 0 ? false : a.lib.num_dofs > 0;
  const int D = robot ? a.lib.num_dofs : 3 * (J - 1);
  const int T = (T_MAX == 1) ? 1 : a.time_steps;
  const int BS = JT > 0 ? round4(JT * kBodyRec) : a.lib.body_stride;
  const StepLayout L = make_layout(J, T, BS, amp_dim, obs_dim, alias_obs, robot ? D : 0);
  float* const w_base = smem + (size_t)warp * L.total;
  float* const s_rslots = w_base;
  float* const s_state = s_rslots + L.rslots;
  float* const s_oslots = s_state + L.state;
  float* const s_dof = s_oslots + L.oslots;
  float* const s_amp = s_dof + L.dof;
  float* const s_obs = alias_obs ? w_base : (s_amp + L.amp);
  uint64_t* const bar = reinterpret_cast<uint64_t*>(w_base + L.total - 4);     // state + reward-time reference
  uint64_t* const bar_o = bar + 1;                                             // observation bracket(s)
  const bool from_cache = (flags & PHC_FLAG_REWARD_FROM_CACHE) && !obs_only;

  // The simulator block (and the cached reference pose) depend only on the env index: their TMA copies are issued before
  // anything else, so this DRAM round trip overlaps the scalar loads -> bracket -> frame-copy chain below.
  const float* g_state = a.body_state + (size_t)env * a.bodies_per_env * kBodyRec;
  const uint32_t state_bytes = (uint32_t)(J * kBodyRec) * 4u;
  const uint32_t frame_bytes = (uint32_t)BS * 4u;
  if (lane == 0) {
    mbar_init(bar, 1);
    mbar_init(bar_o, 1);
    mbar_init_fence();
  }
  // Programmatic dependent launch: everything above (CTA placement, shared-memory carve-up, barrier setup) may run while the
  // previous kernel of the stream is still finishing; no global memory is touched before this wait returns (= the previous
  // grid has completed and its writes are visible).  A no-op when the launch carries no programmatic dependency.
  grid_dependency_wait();
  PHC_TL(0);
  auto issue_env_blocks = [&]() {
    if (lane == 0) {
      if (state_bulk_ok) {
        mbar_expect_tx(bar, state_bytes);
        bulk_g2s(s_state, g_state, state_bytes, bar);
      }
      if (from_cache) {
        mbar_expect_tx(bar, frame_bytes);
        bulk_g2s(s_rslots, a.ref_cache + (size_t)env * BS, frame_bytes, bar);
        mbar_arrive(bar);                  // nothing else lands on this barrier (else: arrive once the reward frames are issued)
      }
    }
    __syncwarp();
  };
  issue_env_blocks();

  // ---- every load that depends only on the env index is issued first (one DRAM round trip for all of them) ----------
  const int64_t progress = a.progress[env];
  // PHC_FLAG_RECOVERY: _update_recovery_count (humanoid_im_getup.py:198-201) -- the counter after this step's decrement.  An env still
  // recovering keeps progress - 1 (:209), which is also the progress its observation is built for (humanoid.py:1641-1647)
  int rcnt = 0;
  if (REC && (flags & PHC_FLAG_RECOVERY)) { const int c = a.recovery_counter[env]; rcnt = c - 1 < 0 ? 0 : c - 1; }
  const int64_t progress_o = (REC && rcnt > 0) ? progress - 1 : progress;
  const float t_start = a.start_times[env], t_off = a.start_offsets[env];
  const V3 goff = v3(a.global_offset[3 * env + 0], a.global_offset[3 * env + 1], a.global_offset[3 * env + 2]);
  float m_len, m_dt;
  int64_t m_nf, m_start;
  if (FAST || a.env_motion) {                         // pre-gathered per-env record: no motion_ids -> table dependency
    const int4 em = *reinterpret_cast<const int4*>(a.env_motion + env);
    m_len = __int_as_float(em.x); m_dt = __int_as_float(em.y); m_nf = em.z; m_start = em.w;
  } else {
    const int64_t mid = a.motion_ids[env];
    m_len = a.lib.motion_len[mid]; m_dt = a.lib.motion_dt[mid];
    m_nf = a.lib.motion_num_frames[mid]; m_start = a.lib.length_starts[mid];
  }
  const float2* g_dof = reinterpret_cast<const float2*>(a.dof_state) + (size_t)env * D;
  const float* g_force = (FAST || a.dof_force) ? a.dof_force + (size_t)env * D : nullptr;
  float2 dof_pv[3];                                   // D <= 93 for J <= 32: at most 3 dofs per lane
  float dof_f[3];
#pragma unroll
  for (int u = 0; u < 3; ++u) {
    const int d = lane + 32 * u;
    dof_pv[u] = (d < D) ? g_dof[d] : make_float2(0.f, 0.f);
    dof_f[u] = (g_force && d < D) ? g_force[d] : 0.f;
  }

  // Motion parameters of the OBSERVATION time: the step's own, unless the clip wraps this step (cycle_motion) -- then the
  // reward still reads the old clip position while the observation (and every later step) follows the re-based one.
  float t_start_o = t_start, t_off_o = t_off;
  V3 goff_o = goff;
  const bool zof = GETUP && (flags & PHC_FLAG_ZERO_OUT_FAR);
  const bool cyc = GETUP && (flags & PHC_FLAG_CYCLE_MOTION) && !obs_only;
  int cc = 0;                                        // _cycle_counter as the reset test sees it
  bool rebased = false;                              // the clip wrapped this step
  if (GETUP) {
    if (a.cycle_counter) cc = a.cycle_counter[env];
    if (cyc) {
      cc = cc - 1 < 0 ? 0 : cc - 1;                  // _update_cycle_count of pre_physics_step (humanoid_im.py:1076-1079)
      const float t_now0 = PHC_ADD(PHC_ADD(PHC_MUL((float)progress, a.dt), t_start), t_off);
      if (t_now0 >= m_len) {                         // pass_time_motion_len (humanoid_im.py:1121-1146)
        t_off_o = -PHC_MUL((float)progress, a.dt);   // progress * dt cancels: the clip restarts at the sampled time
        const float grid = 1.0f / 30.0f;             // sample_time_interval (motion_lib_base.py:414-423)
        const long long k = (long long)((a.cycle_phase[env] * m_len) / grid);
        t_start_o = (float)k * grid;
        // get_root_pos_smpl (motion_lib_base.py:522-547): the clip's root at the new start time, no offset
        const Bracket32 b = frame_bracket32(t_start_o, m_len, (int)m_nf, m_dt);
        const float* r0 = a.lib.frames_body + (size_t)(m_start + b.i0) * BS;
        const float* r1 = a.lib.frames_body + (size_t)(m_start + b.i1) * BS;
        const float omb = 1.0f - b.blend;
        goff_o.x = g_state[0] - lerp1(r0[0], r1[0], omb, b.blend);     // _humanoid_root_states[:, :2] = body 0 of the state block
        goff_o.y = g_state[1] - lerp1(r0[1], r1[1], omb, b.blend);
        cc = 60;
        rebased = true;
        __syncwarp();          // every lane has read the old start / offset values before lane 0 replaces them
        if (lane == 0) {
          a.start_times[env] = t_start_o;
          a.start_offsets[env] = t_off_o;
          a.global_offset[3 * env + 0] = goff_o.x;
          a.global_offset[3 * env + 1] = goff_o.y;
        }
      }
      if (lane == 0 && a.cycle_counter) a.cycle_counter[env] = cc;
    }
  }

  // reward / reset use the CURRENT motion time (humanoid_im.py:879), observations the NEXT one (:752)
  float bl_r = 0.f;
  float bl_o[T_MAX];
  const float* po0[T_MAX];     // shared-memory address of frame i0 / i1 of observation sample t
  const float* po1[T_MAX];
  const float* pr0 = s_rslots;
  const float* pr1 = s_rslots + BS;

  // ---- issue the TMA bulk copies: simulator block + the DISTINCT frames of all brackets ---------------------
  // Observation slots are always filled; a later slot whose frame row was already requested aliases the earlier
  // one.  In steady state (30 fps clips, dt = 1/30) the reward bracket is rows (k, k+1) and the observation
  // bracket (k+1, k+2): 3 distinct frames, the reward slot 1 aliases observation slot 0.
  // (Measured: issuing the observation-bracket copies here, before phase A, beats issuing them after phase A -- 19.5 vs
  // 20.5 us at 4096 envs: the self observation alone is too short to cover their DRAM latency.)
  auto issue_frames = [&]() {
    // the reward bracket is only needed when the reward pose is interpolated here (no pose cache, not the obs-only launch)
    const bool need_r = !from_cache && !obs_only;
    Bracket32 br_r;
    br_r.i0 = 0; br_r.i1 = 0; br_r.blend = 0.f;
    if (need_r) {
      const float t_now = PHC_ADD(PHC_ADD(PHC_MUL((float)progress, a.dt), t_start), t_off);   // motion times: never contracted
      br_r = frame_bracket32(t_now, m_len, (int)m_nf, m_dt);
    }
    bl_r = br_r.blend;
    uint32_t tx_o = 0, tx_r = 0;
    int64_t rows_o[2 * T_MAX];
    bool fresh_o[2 * T_MAX];
#pragma unroll
    for (int t = 0; t < T_MAX; ++t) {
      if (t < T) {
        // ((progress + 1) * dt [+ t * traj_dt] + start + offset), humanoid_im.py:744-752
        float tn = PHC_MUL((float)(progress_o + 1), a.dt);
        if (T > 1) tn = PHC_ADD(tn, PHC_MUL((float)t, a.traj_dt));
        tn = PHC_ADD(PHC_ADD(tn, t_start_o), t_off_o);
        const Bracket32 b = frame_bracket32(tn, m_len, (int)m_nf, m_dt);
        bl_o[t] = b.blend;
        rows_o[2 * t] = m_start + b.i0;
        rows_o[2 * t + 1] = m_start + b.i1;
      }
    }
#pragma unroll
    for (int k = 0; k < 2 * T_MAX; ++k) {
      if (k < 2 * T) {
        const float* ptr = s_oslots + k * BS;
        bool dup = false;
#pragma unroll
        for (int p = 0; p < 2 * T_MAX; ++p)          // static indices only: keeps the arrays in registers
          if (p < k && !dup && rows_o[p] == rows_o[k]) { ptr = (p & 1) ? po1[p >> 1] : po0[p >> 1]; dup = true; }
        if (k & 1) po1[k >> 1] = ptr; else po0[k >> 1] = ptr;
        fresh_o[k] = !dup;
        if (!dup) tx_o += frame_bytes;
      }
    }
    const int64_t row_r0 = m_start + br_r.i0, row_r1 = m_start + br_r.i1;
    bool fresh_r0 = need_r, fresh_r1 = fresh_r0;
    if (fresh_r0) {
#pragma unroll
      for (int p = 0; p < 2 * T_MAX; ++p) {
        if (p < 2 * T) {
          const float* ptr = (p & 1) ? po1[p >> 1] : po0[p >> 1];
          if (fresh_r0 && rows_o[p] == row_r0) { pr0 = ptr; fresh_r0 = false; }
          if (fresh_r1 && rows_o[p] == row_r1) { pr1 = ptr; fresh_r1 = false; }
        }
      }
      if (fresh_r1 && row_r1 == row_r0) { pr1 = pr0; fresh_r1 = false; }
      if (fresh_r0) tx_r += frame_bytes;
      if (fresh_r1) tx_r += frame_bytes;
    }

    if (lane == 0) {
      if (!from_cache) {
        if (tx_r) mbar_expect_tx(bar, tx_r);
        if (fresh_r0) bulk_g2s(s_rslots, a.lib.frames_body + (size_t)row_r0 * BS, frame_bytes, bar);
        if (fresh_r1) bulk_g2s(s_rslots + BS, a.lib.frames_body + (size_t)row_r1 * BS, frame_bytes, bar);
        mbar_arrive(bar);
      }
      mbar_arrive_expect_tx(bar_o, tx_o);
#pragma unroll
      for (int k = 0; k < 2 * T_MAX; ++k)
        if (k < 2 * T && fresh_o[k])
          bulk_g2s(s_oslots + k * BS, a.lib.frames_body + (size_t)rows_o[k] * BS, frame_bytes, bar_o);
    }
  };
  issue_frames();
  PHC_TL(1);
  if (!state_bulk_ok) {      // bodies_per_env not a multiple of 4: rows are only 4-byte aligned
    for (int i = lane; i < J * kBodyRec; i += 32) s_state[i] = g_state[i];
  }

  // ---- while the copies fly: dof state / force (power reward + AMP joint inputs) ---------------------------
  float power = 0.0f;
#pragma unroll
  for (int u = 0; u < 3; ++u) {
    const int d = lane + 32 * u;
    if (d < D) {
      s_dof[2 * d] = dof_pv[u].x;
      s_dof[2 * d + 1] = dof_pv[u].y;
      power += fabsf(dof_f[u] * dof_pv[u].y);
    }
  }
  __syncwarp();
  mbar_wait(bar, 0);
  // without the cache the reward bracket may alias observation slots: phase A then needs those copies too
  if (!from_cache && !obs_only) mbar_wait(bar_o, 0);
  PHC_TL(2);
#if defined(PHC_EXP_EXIT) && PHC_EXP_EXIT == 2      // floor experiment: launch + every input landed in shared memory, nothing else
  mbar_wait(bar_o, 0);
  if (dof_pv[0].x + dof_f[0] + power == 123.456f) a.rew[env] = 0.f;
  return;
#endif

  // ================= phase A: everything that reads the reward slots / simulator block =======================
  const bool has_body = lane < J;
  const bool has_ext = E > 0 && lane >= J && lane < J + E;   // robots: lanes J..J+E-1 carry the "extend" bodies (reward only)
  const int j = has_body ? lane : 0;
  const int jr = (has_body || has_ext) ? lane : 0;           // record of the reference pose this lane tracks
  // env.trackBodies: body j is the slot-th of K tracked bodies (task observation, optionally the reward); K = J, slot = j without a subset
  const bool subset = !FAST && a.num_track > 0;
  const int K = subset ? a.num_track : J;
  const int slot = subset ? (has_body ? (int)a.track_slot[j] : -1) : j;
  const bool tracked = has_body && slot >= 0;
  const bool sub_rew = !FAST && (flags & PHC_FLAG_SUBSET_REWARD);
  BodyRec sim = load_body(s_state + (has_ext ? a.ext_parent[lane - J] : j) * kBodyRec);   // stride-13 words: bank-conflict free
  if (has_ext) {   // parent_rot * pos_in_parent + parent_pos, rotation = the parent's (humanoid_im.py:917-919)
    const V3 off = v3(a.ext_pos[lane - J][0], a.ext_pos[lane - J][1], a.ext_pos[lane - J][2]);
    sim.p = qrot(sim.q, off) + sim.p;
  }
  const V3 root_p = v3(s_state[0], s_state[1], s_state[2]);
  const bool has_h = flags & PHC_FLAG_ROOT_HEIGHT_OBS;
  const int base0 = has_h ? 1 : 0;

  // heading frame of the simulated root
  Q4 root_q = q4(s_state[3], s_state[4], s_state[5], s_state[6]);
  if (!(flags & PHC_FLAG_UPRIGHT)) root_q = strip_base_rot(root_q);
  const float heading = heading_angle(root_q);
  const Q4 hq = quat_about_z(heading);
  const Q4 hinv = q4(0.0f, 0.0f, -hq.z, hq.w);     // quat_about_z(-heading): sin is odd, cos even -> the exact conjugate

  if (!obs_only) {   // the reset-path launch writes observations (and the pose cache) only
    // reward + termination against the reference pose at t_now
    float e_pos = 0.f, e_rot = 0.f, e_vel = 0.f, e_ang = 0.f, dist = 0.f;
    {
      const BodyRec ref = from_cache ? load_body(s_rslots + jr * kBodyRec)
                                     : blend_body(pr0 + jr * kBodyRec, pr1 + jr * kBodyRec, bl_r, goff);
      if (!FAST && a.body_pos_gt && has_body) st3(a.body_pos_gt + ((size_t)env * J + j) * 3, ref.p);
      if (has_body || has_ext) {      // position / rotation terms: all J + E bodies; velocity terms: the J simulated ones
        const V3 dp = ref.p - sim.p;
        const float sp = dp.x * dp.x + dp.y * dp.y + dp.z * dp.z;
        e_pos = sp / 3.0f;
        const float ang = quat_angle(qmul(ref.q, qconj(sim.q)));
        e_rot = ang * ang;
        if (has_body) {
          const V3 dv = ref.v - sim.v, dw = ref.w - sim.w;
          e_vel = (dv.x * dv.x + dv.y * dv.y + dv.z * dv.z) / 3.0f;
          e_ang = (dw.x * dw.x + dw.y * dw.y + dw.z * dw.z) / 3.0f;
          dist = sqrtf(sp);
        }
        if (sub_rew && !tracked) { e_pos = 0.f; e_rot = 0.f; e_vel = 0.f; e_ang = 0.f; }   // reward over the tracked subset (the reset test keeps `dist`)
      }
    }
    if (!FAST && a.mpjpe) {        // flags.im_eval extras (humanoid_im.py:674-680): mean per-joint position error + the pose it is against
      const float mp = warp_sum(has_body ? dist : 0.0f) / (float)J;
      if (lane == 0) a.mpjpe[env] = mp;
    }
    float dist_t = dist;           // the distance the termination test sees
    if (!FAST && a.occlusion && has_body && a.occlusion[(size_t)env * K + slot]) dist_t = 0.0f;   // an occluded body cannot fail it (humanoid_im.py:1180-1181)
    if (GETUP && rebased) {
      // the clip wrapped this step: the reference's reset test re-queries the pose at the re-based time (humanoid_im.py:1142,
      // :1148).  Rare (once per clip length): positions straight from the frame table, no staging.
      const float t_re = PHC_ADD(PHC_ADD(PHC_MUL((float)progress, a.dt), t_start_o), t_off_o);
      const Bracket32 b = frame_bracket32(t_re, m_len, (int)m_nf, m_dt);
      const float* r0 = a.lib.frames_body + (size_t)(m_start + b.i0) * BS + jr * kBodyRec;
      const float* r1 = a.lib.frames_body + (size_t)(m_start + b.i1) * BS + jr * kBodyRec;
      const V3 pr = lerp3(v3(r0[0], r0[1], r0[2]), v3(r1[0], r1[1], r1[2]), 1.0f - b.blend, b.blend) + goff_o;
      const V3 d2 = pr - sim.p;
      dist_t = has_body ? sqrtf(d2.x * d2.x + d2.y * d2.y + d2.z * d2.z) : 0.f;
    }
    bool fallen;
    {
      const float thr = has_body ? a.term_thresh[j] : INFINITY;
      if (flags & PHC_FLAG_TERM_USE_MEAN) {
        const bool in_set = has_body && thr < INFINITY;
        const float cnt = warp_sum(in_set ? 1.0f : 0.0f);
        const float sum = warp_sum(in_set ? dist_t : 0.0f);
        fallen = (sum / cnt) > a.term_dist_mean;
      } else {
        fallen = __any_sync(0xffffffffu, has_body && dist_t > thr);
      }
    }
    // the four error sums in one 6-shuffle reduction: lanes 8k..8k+7 end up with sum k, finish "their" reward term
    // exp(-k * mean) (one expf sequence for the warp instead of four on lane 0) and hand it to lane 0
    const float e4 = warp_sum4(e_pos, e_rot, e_vel, e_ang, lane);
    const int sel = lane >> 3;
    const float den = sub_rew ? (float)K : (sel < 2 ? (float)(J + E) : (float)J);
    const float kc = sel == 0 ? a.k_pos : (sel == 1 ? a.k_rot : (sel == 2 ? a.k_vel : a.k_ang_vel));
    const float r_mine = expf(-kc * (e4 / den));
    const float r_pos = __shfl_sync(0xffffffffu, r_mine, 0), r_rot = __shfl_sync(0xffffffffu, r_mine, 8);
    const float r_vel = __shfl_sync(0xffffffffu, r_mine, 16), r_ang = __shfl_sync(0xffffffffu, r_mine, 24);
    power = warp_sum(power);

    if (lane == 0) {
      float rew = a.w_pos * r_pos + a.w_rot * r_rot + a.w_vel * r_vel + a.w_ang_vel * r_ang;
      const bool has_power = flags & PHC_FLAG_POWER_REWARD;
      const int rw = has_power ? 5 : 4;
      float* raw = a.reward_raw + (size_t)env * rw;
      float w0 = r_pos, w1 = r_rot, w2 = r_vel, w3 = r_ang;
      if (zof) {
        // point-goal mix (humanoid_im.py:890-905): lane 0 tracks the root, `dist` is |root_pos - ref_root_pos|.  Everywhere:
        // clamp(previous distance - distance, max = 1/3) * 9; within the 0.25 m transition distance half the imitation reward on top
        const float pg = fminf(a.point_goal[env] - dist, 1.0f / 3.0f) * 9.0f;
        if (dist > 0.25f) { rew = pg; w0 = pg; w1 = 0.0f; w2 = 0.0f; w3 = 0.0f; }
        else { rew = pg + rew * 0.5f; w0 = pg + r_pos * 0.5f; w1 = 0.0f + r_rot * 0.5f; w2 = 0.0f + r_vel * 0.5f; w3 = 0.0f + r_ang * 0.5f; }
      }
      raw[0] = w0; raw[1] = w1; raw[2] = w2; raw[3] = w3;
      if (has_power) {
        float pr = -a.power_coef * power;
        if (progress <= 3) pr = 0.0f;
        rew = rew + pr;
        raw[4] = pr;
      }
      a.rew[env] = rew;
      // compute_humanoid_im_reset + the is_recovery override
      const float t_now = PHC_ADD(PHC_ADD(PHC_MUL((float)progress, a.dt), t_start), t_off);
      bool pass_time = t_now >= m_len;
      if (cyc) pass_time = progress >= (int64_t)a.max_episode_length - 1;      // pass_time_max (humanoid_im.py:1120-1124)
      int64_t terminated = 0;
      if (flags & PHC_FLAG_EARLY_TERM) {
        bool f = fallen && (progress > 1);
        if (flags & PHC_FLAG_NO_COLLISION) f = false;
        terminated = f ? 1 : 0;
      }
      int64_t reset = pass_time ? 1 : terminated;
      if (GETUP) { if (!pass_time && cc > 0) { reset = 0; terminated = 0; } }
      else if (a.cycle_counter && !pass_time && a.cycle_counter[env] > 0) { reset = 0; terminated = 0; }
      if (REC && rcnt > 0) { reset = 0; terminated = 0; }      // humanoid_im_getup.py:203-210: not cancelled by pass_time
      a.reset[env] = reset;
      a.terminate[env] = terminated;
    }
  }

  // AMP observation of the simulated character (build_amp_observations_smpl) -> its own staging row; the observation-only launch
  // writes it only with PHC_FLAG_AMP_CURRENT (the get-up reset path)
  const bool amp_cur = REC && obs_only && (flags & PHC_FLAG_AMP_CURRENT);
  if ((FAST || a.amp_out) && (!obs_only || amp_cur)) {
    const int nj = a.num_amp_joints, nk = a.num_key_bodies;
    float* o = s_amp + base0;
    if (lane == 0) {
      if (has_h) s_amp[0] = root_p.z;
      // root columns: with an upright start they ARE the self observation's root entries (same heading frame, same
      // rotation) and are copied from there in phase B; only the remove_base_rot case differs (humanoid_amp.py:980-982)
      if (!(flags & PHC_FLAG_UPRIGHT)) {
        st6(o, tan_norm((flags & PHC_FLAG_LOCAL_ROOT_OBS) ? qmul_zl(hinv, root_q) : root_q));
        st3(o + 6, qrot_z(hinv, sim.v));      // lane 0 holds body 0 = the root
        st3(o + 9, qrot_z(hinv, sim.w));
      }
    }
    if (robot) {       // build_amp_observations_robot (humanoid_amp.py:1062-1104): raw hinge angles, then velocities
      for (int d = lane; d < D; d += 32) { o[12 + d] = s_dof[2 * d]; o[12 + D + d] = s_dof[2 * d + 1]; }
    }
    for (int k = lane; k < (robot ? 0 : nj); k += 32) {
      const int jid = a.amp_joints[k];
      const float* dj = s_dof + 6 * jid;             // (pos, vel) pairs of the joint's 3 dofs
      st6(o + 12 + 6 * k, tan_norm(exp_map_to_quat(v3(dj[0], dj[2], dj[4]))));
      st3(o + 12 + 6 * nj + 3 * k, v3(dj[1], dj[3], dj[5]));
    }
    if (lane < nk) {
      const float* kb = s_state + a.key_bodies[lane] * kBodyRec;
      st3(o + 12 + (robot ? 2 * D : 9 * nj) + 3 * lane, qrot_z(hinv, v3(kb[0], kb[1], kb[2]) - root_p));
    }
  }
  // rows leave shared memory as TMA bulk stores (one instruction per row) when source, destination and size are 16-byte
  // granular; otherwise with per-lane coalesced stores; all rows of the env go out together at the end.
  // ring mode with the head on the device (PhcStepArgs.ring_head): this step's vector goes to slot *ring_head of the env's ring
  float* const g_amp = ((FAST || a.amp_out) && (!obs_only || amp_cur))
                           ? a.amp_out + (size_t)env * a.amp_out_stride + (a.ring_head ? (size_t)(*a.ring_head) * (size_t)amp_dim : (size_t)0) : nullptr;
  const bool amp_bulk = FAST ? true : (g_amp && !a.amp_hist_in && (amp_dim & 3) == 0 && (reinterpret_cast<uintptr_t>(g_amp) & 15) == 0);
  __syncwarp();   // the reward slots and the simulator block are consumed: the obs row may overwrite them
  PHC_TL(3);
  if (REC && (flags & PHC_FLAG_RECOVERY) && lane == 0) {     // every lane has read both values: write them back
    a.recovery_counter[env] = rcnt;
    if (rcnt > 0) const_cast<int64_t*>(a.progress)[env] = progress_o;
  }

  // ================= phase B: observation row (reads only registers + the observation slots) =================
  if (lane == 0 && has_h) s_obs[0] = root_p.z;
  if (has_body) {
    // self observation (compute_humanoid_observations_smpl_max)
    float* o_pos = s_obs + base0;
    float* o_rot = o_pos + 3 * (J - 1);
    float* o_vel = o_rot + 6 * J;
    float* o_ang = o_vel + 3 * J;
    if (j > 0) st3(o_pos + 3 * (j - 1), qrot_z(hinv, sim.p - root_p));
    TanNorm tn = tan_norm(qmul_zl(hinv, sim.q));
    if (j == 0 && !(flags & PHC_FLAG_LOCAL_ROOT_OBS)) tn = tan_norm(root_q);
    const V3 lv = qrot_z(hinv, sim.v), lw = qrot_z(hinv, sim.w);
    st6(o_rot + 6 * j, tn);
    st3(o_vel + 3 * j, lv);
    st3(o_ang + 3 * j, lw);
    if (j == 0 && (FAST || g_amp) && (flags & PHC_FLAG_UPRIGHT)) {     // AMP root columns = the root's self-observation entries
      float* o = s_amp + base0;
      st6(o, tn); st3(o + 6, lv); st3(o + 9, lw);
    }
  }
  if (!FAST && (a.shape_params || a.limb_weights)) {          // has_shape_obs / has_limb_weight_obs columns (humanoid.py:2043-2047)
    float* o_ext = s_obs + base0 + 15 * J - 3;
    const int ns = a.shape_params ? a.num_shape : 0, nl = a.limb_weights ? a.num_limb : 0;
    for (int c = lane; c < ns; c += 32) o_ext[c] = a.shape_params[(size_t)env * ns + c];
    for (int c = lane; c < nl; c += 32) o_ext[ns + c] = a.limb_weights[(size_t)env * nl + c];
  }
  // task observation (v6, or v7 with KP) for each of the T reference samples (the self observation above did not need the frames)
  mbar_wait(bar_o, 0);
  PHC_TL(4);
  float* const g_cache = (FAST || a.ref_cache) ? a.ref_cache + (size_t)env * BS : nullptr;
  const bool cache_bulk = FAST ? true : (g_cache && T_MAX == 1);     // single sample: the blended pose is staged over its own frame slot
  V3 rroot = v3(0.f, 0.f, 0.f);
  if (zof) {
    // zero_out_far needs |root_pos - reference root| in every lane: each lane blends the reference ROOT position itself (the
    // same shared-memory words for all lanes: a broadcast read, bit-identical to lane 0's blend_body) ...
    const float* s0 = po0[0];
    const float* s1 = po1[0];
    rroot = lerp3(v3(s0[0], s0[1], s0[2]), v3(s1[0], s1[1], s1[2]), 1.0f - bl_o[0], bl_o[0]) + goff_o;
    __syncwarp();      // ... before lane 0 may overwrite record 0 of the slot with the cached pose
  }
#pragma unroll
  for (int t = 0; t < T_MAX; ++t) {
    if (t < T && (has_body || (has_ext && t == 0 && (FAST || g_cache)))) {
      const BodyRec ref = blend_body(po0[t] + jr * kBodyRec, po1[t] + jr * kBodyRec, bl_o[t], goff_o);
      if (t == 0 && (FAST || g_cache)) {
        // lane j has consumed records j of both frames: slot 0 of the bracket becomes the row of the pose cache
        float* c = (cache_bulk ? s_oslots : g_cache) + jr * kBodyRec;
        st3(c, ref.p); c[3] = ref.q.x; c[4] = ref.q.y; c[5] = ref.q.z; c[6] = ref.q.w; st3(c + 7, ref.v); st3(c + 10, ref.w);
      }
      if (!has_body) continue;         // extend bodies: reward only, no observation columns
      if (t == 0) {     // side buffers of _compute_task_obs(save_buffer=True): every body, tracked or not
        const size_t bj = (size_t)env * J + j;
        if (!FAST && a.ref_body_pos) st3(a.ref_body_pos + 3 * bj, ref.p);
        if (!FAST && a.ref_body_vel) st3(a.ref_body_vel + 3 * bj, ref.v);
        if (!FAST && a.ref_body_ang_vel) st3(a.ref_body_ang_vel + 3 * bj, ref.w);
        if (!FAST && a.ref_body_rot) { float* d = a.ref_body_rot + 4 * bj; d[0] = ref.q.x; d[1] = ref.q.y; d[2] = ref.q.z; d[3] = ref.q.w; }
      }
      if (!tracked) continue;          // env.trackBodies: only the tracked bodies have task-observation columns
      BodyRec ro = ref;                // what the observation sees as reference (the cache / ref_* buffers keep `ref`)
      if (zof && t == 0) {             // humanoid_im.py:783-796 (v7: :834-845, the same overwrites of the columns it has)
        const V3 dr = root_p - rroot;
        const float dist = sqrtf(dr.x * dr.x + dr.y * dr.y + dr.z * dr.z);
        if (dist > a.close_distance) {       // far from the reference: it collapses onto the simulated pose (root position excepted)
          if (j > 0) { ro.p = sim.p; ro.q = sim.q; }
          ro.v = sim.v; ro.w = sim.w;
        }
        if (dist > a.far_distance && j == 0)   // very far: the root target becomes a direction of length far_distance
          ro.p = v3((ref.p.x - sim.p.x) / dist * a.far_distance + sim.p.x, (ref.p.y - sim.p.y) / dist * a.far_distance + sim.p.y,
                    (ref.p.z - sim.p.z) / dist * a.far_distance + sim.p.z);
        if (lane == 0) a.point_goal[env] = dist;
      }
      if (!FAST && a.occlusion && t == 0 && a.occlusion[(size_t)env * K + slot]) {   // _occl_training (humanoid_im.py:797-804)
        ro.p = sim.p; ro.q = sim.q;
        if (!KP) { ro.v = sim.v; ro.w = sim.w; }      // v7 (:847-851) keeps the reference velocity of an occluded body
      }
      if (KP) {         // compute_imitation_observations_v7 (humanoid_im.py:1362-1393): [diff_pos | diff_vel | ref_pos - root] per sample
        float* tb = s_obs + self_dim + t * 9 * K;
        st3(tb + 3 * slot, qrot_z(hinv, ro.p - sim.p));
        st3(tb + 3 * K + 3 * slot, qrot_z(hinv, ro.v - sim.v));
        st3(tb + 6 * K + 3 * slot, qrot_z(hinv, ro.p - root_p));
        continue;
      }
      float* tb = s_obs + self_dim + t * 24 * K;
      st3(tb + 3 * slot, qrot_z(hinv, ro.p - sim.p));
      st6(tb + 3 * K + 6 * slot, tan_norm(qmul_zr(qmul_zl(hinv, qmul(ro.q, qconj(sim.q))), hq)));
      st3(tb + 9 * K + 3 * slot, qrot_z(hinv, ro.v - sim.v));
      st3(tb + 12 * K + 3 * slot, qrot_z(hinv, ro.w - sim.w));
      st3(tb + 15 * K + 3 * slot, qrot_z(hinv, ro.p - root_p));
      st6(tb + 18 * K + 6 * slot, tan_norm(qmul_zl(hinv, ro.q)));
    }
  }
  // ---- rows leave shared memory ---------------------------------------------------------------------------------
  float* const g_obs = a.obs + (size_t)env * a.obs_stride;
  const int obs_pad = round4(obs_dim);
  const bool obs_bulk = FAST ? true : (a.obs_stride >= obs_pad && (reinterpret_cast<uintptr_t>(g_obs) & 15) == 0);
  if (obs_bulk && lane < obs_pad - obs_dim) s_obs[obs_dim + lane] = 0.f;      // the row's pad columns are written as zeros
  if (obs_bulk || cache_bulk || amp_bulk) fence_async_smem();
  __syncwarp();
  PHC_TL(5);
  if (lane == 0 && (obs_bulk || cache_bulk || amp_bulk)) {
    if (amp_bulk) bulk_s2g(g_amp, s_amp, (uint32_t)amp_dim * 4u);
    if (obs_bulk) bulk_s2g(g_obs, s_obs, (uint32_t)obs_pad * 4u);
    if (cache_bulk) bulk_s2g(g_cache, s_oslots, frame_bytes);
    bulk_commit();
  }
  if (obs_bulk) {
  } else if (((a.obs_stride | (int64_t)obs_dim) & 1) == 0) {      // rows 8-byte aligned: float2 stores
    float2* g2 = reinterpret_cast<float2*>(g_obs);
    const float2* s2 = reinterpret_cast<const float2*>(s_obs);
#pragma unroll 5
    for (int i = lane; i < obs_dim / 2; i += 32) g2[i] = s2[i];
  } else {
    for (int i = lane; i < obs_dim; i += 32) g_obs[i] = s_obs[i];
  }
  if (g_amp && !amp_bulk) {
    if (a.amp_hist_in) {
      // newest-first window shift: slot s -> s+1, walking from the oldest slot so an in-place shift is safe
      // (each element is read and later overwritten by the SAME lane, program order keeps it correct)
      const float* h = a.amp_hist_in + (size_t)env * a.amp_out_stride;
      for (int s = a.amp_steps - 2; s >= 0; --s)
        for (int i = lane; i < amp_dim; i += 32) g_amp[(size_t)(s + 1) * amp_dim + i] = h[(size_t)s * amp_dim + i];
    }
#pragma unroll 7
    for (int i = lane; i < amp_dim; i += 32) g_amp[i] = s_amp[i];
  }
  // the shared-memory rows must outlive the bulk reads: the issuing lane waits before the warp (and so the CTA) may retire
  if (lane == 0 && (amp_bulk || obs_bulk || cache_bulk)) bulk_wait_read0();
  PHC_TL(6);
}

}  // namespace phc

// ------------------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------------------
extern "C" void phc_set_error(const char* msg);   // phc_api.cu
extern "C" int phc_check_cuda(cudaError_t e, const char* what);
extern "C" void phc_count_launches(int n);
extern "C" int phc_env_step_wide_launch(const PhcStepArgs* a, int obs_dim, int self_dim, int amp_dim, void* stream);   // env_step_wide.cu
extern "C" int phc_env_step_fast_launch(const PhcStepArgs* a, int amp_dim, int pdl, void* stream);                      // env_step_fast.cu

extern "C" int phc_self_obs_dim(int32_t J, uint32_t flags) {
  return ((flags & PHC_FLAG_ROOT_HEIGHT_OBS) ? 1 : 0) + 15 * J - 3;
}
extern "C" int phc_task_obs_dim(int32_t J, int32_t T) { return 24 * J * T; }
extern "C" int phc_task_obs_dim_flags(int32_t J, int32_t T, uint32_t flags) { return ((flags & PHC_FLAG_TASK_OBS_KP) ? 9 : 24) * J * T; }
extern "C" int phc_amp_obs_dim(int32_t nj, int32_t nk, uint32_t flags) {
  return ((flags & PHC_FLAG_ROOT_HEIGHT_OBS) ? 1 : 0) + 12 + 9 * nj + 3 * nk;
}
extern "C" int phc_amp_obs_dim_robot(int32_t D, int32_t nk, uint32_t flags) {
  return ((flags & PHC_FLAG_ROOT_HEIGHT_OBS) ? 1 : 0) + 12 + 2 * D + 3 * nk;
}

#ifdef PHC_EXP_TIMELINE
extern "C" PHC_API int phc_exp_set_timeline(void* buf) {
  unsigned long long* p = static_cast<unsigned long long*>(buf);
  return phc_check_cuda(cudaMemcpyToSymbol(phc::g_timeline, &p, sizeof(p)), "phc_exp_set_timeline");
}
#endif

static int64_t g_fast_launches = 0;
extern "C" int64_t phc_env_step_fast_launches(void) { return g_fast_launches; }

extern "C" int phc_env_step(const PhcStepArgs* a, void* stream) {
  using namespace phc;
  if (!a) { phc_set_error("phc_env_step: args is NULL"); return PHC_ERR_INVALID_ARG; }
  if (a->num_envs == 0) return PHC_OK;
  const int J = a->lib.num_bodies, T = a->time_steps;
  if (!a->body_state || !a->dof_state || !a->progress || !a->motion_ids || !a->start_times || !a->start_offsets ||
      !a->global_offset || !a->lib.frames_body || !a->lib.motion_len || !a->lib.motion_dt ||
      !a->lib.motion_num_frames || !a->lib.length_starts || !a->obs ||
      (!(a->flags & PHC_FLAG_OBS_ONLY) && (!a->rew || !a->reward_raw || !a->reset || !a->terminate))) {
    phc_set_error("phc_env_step: a required pointer is NULL");
    return PHC_ERR_INVALID_ARG;
  }
  if (a->num_envs < 0 || J < 1 || a->bodies_per_env < J || T < 1) {
    phc_set_error("phc_env_step: bad sizes (num_envs >= 0, 1 <= J <= bodies_per_env, T >= 1)");
    return PHC_ERR_INVALID_ARG;
  }
  const int E = a->lib.num_ext_bodies, DR = a->lib.num_dofs;
  if (E < 0 || E > PHC_MAX_EXT_BODIES || DR < 0) { phc_set_error("phc_env_step: bad num_ext_bodies / num_dofs"); return PHC_ERR_INVALID_ARG; }
  if (J + E > PHC_MAX_BODIES) { phc_set_error("phc_env_step: more than PHC_MAX_BODIES bodies (incl. extend bodies)"); return PHC_ERR_UNSUPPORTED; }
  const bool wide = J + E > PHC_LANE_BODIES || DR > 3 * PHC_LANE_BODIES;      // strided kernel of env_step_wide.cu
  for (int e2 = 0; e2 < E; ++e2)
    if (a->ext_parent[e2] < 0 || a->ext_parent[e2] >= J) { phc_set_error("phc_env_step: ext_parent out of range"); return PHC_ERR_INVALID_ARG; }
  if (T > 4) { phc_set_error("phc_env_step: time_steps > 4 not supported"); return PHC_ERR_UNSUPPORTED; }
  const bool getup = (a->flags & (PHC_FLAG_ZERO_OUT_FAR | PHC_FLAG_CYCLE_MOTION)) != 0;
  if (getup) {
    if (T != 1 || E != 0 || DR != 0) { phc_set_error("phc_env_step: zero_out_far / cycle_motion are built for time_steps 1 and spherical-joint humanoids"); return PHC_ERR_UNSUPPORTED; }
    if ((a->flags & PHC_FLAG_ZERO_OUT_FAR) && (!a->point_goal || !(a->far_distance > 0.0f))) { phc_set_error("phc_env_step: zero_out_far needs point_goal and far_distance > 0"); return PHC_ERR_INVALID_ARG; }
    if ((a->flags & PHC_FLAG_CYCLE_MOTION) && (!a->cycle_phase || !a->cycle_counter || a->max_episode_length < 1)) {
      phc_set_error("phc_env_step: cycle_motion needs cycle_phase, cycle_counter and max_episode_length >= 1"); return PHC_ERR_INVALID_ARG;
    }
  }
  if ((a->flags & PHC_FLAG_POWER_REWARD) && !a->dof_force) { phc_set_error("phc_env_step: power reward needs dof_force"); return PHC_ERR_INVALID_ARG; }
  if (a->num_key_bodies < 0 || a->num_key_bodies > PHC_MAX_KEY_BODIES || a->num_amp_joints < 0 || a->num_amp_joints > PHC_MAX_AMP_JOINTS) {
    phc_set_error("phc_env_step: bad key body / amp joint lists"); return PHC_ERR_INVALID_ARG;
  }
  if (a->lib.body_stride != phc_motion_body_stride(J + E) || (reinterpret_cast<uintptr_t>(a->lib.frames_body) & 15)) {
    phc_set_error("phc_env_step: frames_body must be 16-byte aligned with body_stride = round_up(13*(J+E),4) (use phc_motion_pack)");
    return PHC_ERR_INVALID_ARG;
  }
  if (a->env_motion && (reinterpret_cast<uintptr_t>(a->env_motion) & 15)) { phc_set_error("phc_env_step: env_motion must be 16-byte aligned"); return PHC_ERR_INVALID_ARG; }
  if (reinterpret_cast<uintptr_t>(a->dof_state) & 7) { phc_set_error("phc_env_step: dof_state must be 8-byte aligned"); return PHC_ERR_INVALID_ARG; }
  const int n_shape = a->shape_params ? a->num_shape : 0, n_limb = a->limb_weights ? a->num_limb : 0;
  if (a->num_track < 0 || a->num_track > J || n_shape < 0 || n_limb < 0) { phc_set_error("phc_env_step: bad num_track / num_shape / num_limb"); return PHC_ERR_INVALID_ARG; }
  if (a->num_track > 0) {
    int seen = 0;
    for (int b = 0; b < J; ++b) if (a->track_slot[b] >= 0) { if (a->track_slot[b] >= a->num_track) { phc_set_error("phc_env_step: track_slot out of range"); return PHC_ERR_INVALID_ARG; } ++seen; }
    if (seen != a->num_track) { phc_set_error("phc_env_step: track_slot must name exactly num_track bodies"); return PHC_ERR_INVALID_ARG; }
  }
  if (a->occlusion && a->num_track > 0) { phc_set_error("phc_env_step: occlusion training needs every body tracked (the reference indexes random_occlu_idx by body id, humanoid_im.py:1181)"); return PHC_ERR_UNSUPPORTED; }
  const bool kp = (a->flags & PHC_FLAG_TASK_OBS_KP) != 0;
  if (kp && wide) { phc_set_error("phc_env_step: the keypoint task observation (PHC_FLAG_TASK_OBS_KP) is built for <= 32-body humanoids"); return PHC_ERR_UNSUPPORTED; }
  if (kp && getup && J != 24) { phc_set_error("phc_env_step: the keypoint task observation with zero_out_far / cycle_motion is built for 24-body SMPL"); return PHC_ERR_UNSUPPORTED; }
  // get-up schedule (PHC_FLAG_RECOVERY on a step launch, PHC_FLAG_AMP_CURRENT on the observation-only one): the GETUP instantiations
  const bool recovery = (a->flags & PHC_FLAG_RECOVERY) != 0, amp_cur = (a->flags & PHC_FLAG_AMP_CURRENT) != 0;
  const bool obs_only_l = (a->flags & PHC_FLAG_OBS_ONLY) != 0;
  if (recovery && obs_only_l) { phc_set_error("phc_env_step: PHC_FLAG_RECOVERY is for step launches, not the observation-only launch"); return PHC_ERR_INVALID_ARG; }
  if (recovery && !a->recovery_counter) { phc_set_error("phc_env_step: PHC_FLAG_RECOVERY needs recovery_counter"); return PHC_ERR_INVALID_ARG; }
  if (amp_cur && (!obs_only_l || !a->amp_out)) { phc_set_error("phc_env_step: PHC_FLAG_AMP_CURRENT needs PHC_FLAG_OBS_ONLY and amp_out"); return PHC_ERR_INVALID_ARG; }
  if ((recovery || amp_cur) && (T != 1 || E != 0 || DR != 0)) {
    phc_set_error("phc_env_step: the get-up schedule (PHC_FLAG_RECOVERY / PHC_FLAG_AMP_CURRENT) is built for time_steps 1 and spherical-joint humanoids without extend bodies");
    return PHC_ERR_UNSUPPORTED;
  }
  if ((recovery || amp_cur) && kp && J != 24) { phc_set_error("phc_env_step: the keypoint task observation with the get-up schedule is built for 24-body SMPL"); return PHC_ERR_UNSUPPORTED; }
  const bool widened = a->num_track > 0 || a->occlusion || n_shape > 0 || n_limb > 0 || (a->flags & PHC_FLAG_SUBSET_REWARD);
  if (widened && (wide || E > 0)) { phc_set_error("phc_env_step: tracked-body subsets / occlusion / shape columns are built for <= 32-body humanoids without extend bodies"); return PHC_ERR_UNSUPPORTED; }
  const int self_dim = phc_self_obs_dim(J, a->flags) + n_shape + n_limb;
  const int obs_dim = self_dim + phc_task_obs_dim_flags(a->num_track > 0 ? a->num_track : J, T, a->flags);
  const int amp_dim = !a->amp_out ? 0 : (DR > 0 ? phc_amp_obs_dim_robot(DR, a->num_key_bodies, a->flags)
                                                 : phc_amp_obs_dim(a->num_amp_joints, a->num_key_bodies, a->flags));
  if (a->obs_stride < obs_dim) { phc_set_error("phc_env_step: obs_stride smaller than the observation"); return PHC_ERR_INVALID_ARG; }
  if (a->amp_out && (a->amp_steps < 1 || a->amp_out_stride < (int64_t)(a->amp_hist_in ? a->amp_steps : 1) * amp_dim)) {
    phc_set_error("phc_env_step: amp_out_stride / amp_steps inconsistent"); return PHC_ERR_INVALID_ARG;
  }
  if (wide) return phc_env_step_wide_launch(a, obs_dim, self_dim, amp_dim, stream);
  // the obs row is staged over [reward slots | simulator block] when it fits (always for T == 1)
  const bool alias_obs = (2 * a->lib.body_stride + round4(J * kBodyRec) >= round4(obs_dim));   // incl. the row pad
  const bool obs_row_aligned = ((reinterpret_cast<uintptr_t>(a->obs) & 7) == 0);
  if (!obs_row_aligned) { phc_set_error("phc_env_step: obs must be 8-byte aligned"); return PHC_ERR_INVALID_ARG; }
  // TMA bulk copy of the per-env simulator block needs 16-byte aligned rows of a multiple of 16 bytes
  const bool state_bulk_ok = ((reinterpret_cast<uintptr_t>(a->body_state) & 15) == 0) &&
                             ((a->bodies_per_env * kBodyRec) % 4 == 0) && ((J * kBodyRec) % 4 == 0);
  const StepLayout L = make_layout(J, T, a->lib.body_stride, amp_dim, obs_dim, alias_obs, DR);
  const size_t smem = (size_t)kWarpsPerCta * L.total * sizeof(float);
  const int grid = (a->num_envs + kWarpsPerCta - 1) / kWarpsPerCta;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e;
#define PHC_LAUNCH_STEP(TM, JJ, ...)                                                                                 \
  do {                                                                                                               \
    static size_t smem_limit = 48 * 1024;     /* default opt-out limit; the attribute is only ever RAISED */          \
    if (smem > smem_limit) {                                                                                         \
      e = cudaFuncSetAttribute(env_step_kernel<TM, JJ, __VA_ARGS__>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
      if (e != cudaSuccess) return phc_check_cuda(e, "cudaFuncSetAttribute(env_step_kernel)");                       \
      smem_limit = smem;                                                                                             \
    }                                                                                                                \
    cudaLaunchConfig_t lc = {};                                                                                      \
    lc.gridDim = dim3((unsigned)grid); lc.blockDim = dim3(kWarpsPerCta * 32); lc.dynamicSmemBytes = smem; lc.stream = st; \
    cudaLaunchAttribute la[1];                                                                                       \
    la[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                                   \
    la[0].val.programmaticStreamSerializationAllowed = 1;                                                            \
    lc.attrs = la; lc.numAttrs = pdl_allowed ? 1 : 0;                                                                \
    e = cudaLaunchKernelEx(&lc, env_step_kernel<TM, JJ, __VA_ARGS__>, *a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); \
    if (e != cudaSuccess) return phc_check_cuda(e, "cudaLaunchKernelEx(env_step_kernel)");                           \
    phc_count_launches(1);                                                                                           \
  } while (0)
  // the steady-state launch of the shipped SMPL configuration takes the compile-time specialisation (see kFastFlags)
  const int obs_pad_h = round4(obs_dim);
  // PHC_ENV_PDL=0: plain stream-ordered launches (A/B switch; the kernel's griddepcontrol.wait is then a no-op)
  static const bool pdl_allowed = [] { const char* v = getenv("PHC_ENV_PDL"); return !(v && v[0] == '0'); }();
  static const bool fast_allowed = [] { const char* v = getenv("PHC_ENV_FAST"); return !(v && v[0] == '0'); }();   // A/B switch
  const bool fast = fast_allowed && !widened && !getup && T == 1 && J == 24 && E == 0 && DR == 0 && a->flags == kFastFlags && !a->only_where && a->env_motion &&
                    a->dof_force && state_bulk_ok && alias_obs && a->ref_cache && (reinterpret_cast<uintptr_t>(a->ref_cache) & 15) == 0 &&
                    !a->ref_body_pos && !a->ref_body_rot && !a->ref_body_vel && !a->ref_body_ang_vel &&
                    a->amp_out && !a->amp_hist_in && (amp_dim & 3) == 0 && (reinterpret_cast<uintptr_t>(a->amp_out) & 15) == 0 &&
                    (a->amp_out_stride & 3) == 0 && (reinterpret_cast<uintptr_t>(a->obs) & 15) == 0 && a->obs_stride >= obs_pad_h &&
                    (a->obs_stride & 3) == 0 && a->num_key_bodies > 0;
  // ... in the form of env_step_fast.cu (the same arithmetic with the phases ordered by input arrival); PHC_ENV_FASTK=0 keeps the
  // FAST instantiation of the kernel above (A/B switch, bit-identity tests)
  static const bool fastk_allowed = [] { const char* v = getenv("PHC_ENV_FASTK"); return !(v && v[0] == '0'); }();
  if (fast && fastk_allowed && a->num_amp_joints <= 32 && obs_dim == 934) {
    ++g_fast_launches;
    return phc_env_step_fast_launch(a, amp_dim, pdl_allowed ? 1 : 0, stream);
  }
  if (recovery || amp_cur) {      // the flags are not in kFastFlags: get-up launches never take the FAST paths
    if (kp) PHC_LAUNCH_STEP(1, 24, true, false, true, true);
    else if (J == 24) PHC_LAUNCH_STEP(1, 24, true, false, false, true);
    else PHC_LAUNCH_STEP(1, 0, true, false, false, true);
  }
  else if (kp) {            // PHC_FLAG_TASK_OBS_KP is not in kFastFlags: keypoint launches never take the FAST paths
    if (getup) PHC_LAUNCH_STEP(1, 24, true, false, true);
    else if (T == 1 && J == 24 && E == 0 && DR == 0) PHC_LAUNCH_STEP(1, 24, false, false, true);
    else if (T == 1) PHC_LAUNCH_STEP(1, 0, false, false, true);
    else PHC_LAUNCH_STEP(4, 0, false, false, true);
  }
  else if (fast) { PHC_LAUNCH_STEP(1, 24, false, true); ++g_fast_launches; }
  else if (getup && J == 24) PHC_LAUNCH_STEP(1, 24, true);                      // env_im_getup_mcp.yaml
  else if (getup) PHC_LAUNCH_STEP(1, 0, true);
  else if (T == 1 && J == 24 && E == 0 && DR == 0) PHC_LAUNCH_STEP(1, 24, false);   // SMPL
  else if (T == 1) PHC_LAUNCH_STEP(1, 0, false);                                // H1 (J = 20, E = 3, 19 hinge dofs) and others
  else PHC_LAUNCH_STEP(4, 0, false);
#undef PHC_LAUNCH_STEP
  return phc_check_cuda(cudaGetLastError(), "env_step_kernel launch");
}
