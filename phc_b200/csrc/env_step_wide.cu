// Fused post-physics env step for characters with MORE THAN 32 bodies (incl. extend bodies): Unitree G1 (38 + 1, 37 hinge
// dofs, phc/data/cfg/robot/unitree_g1.yaml) and SMPL-X (52 bodies, phc/data/cfg/robot/smplx_humanoid.yaml).  Same entry point
// and the same semantics as env_step.cu (phc_env_step dispatches here when J + E > 32): reward + reset at the current motion
// time, self + task observation v6 (T <= 4 future samples) at the next one, AMP observation (+ window shift), pose cache,
// ref_* side buffers, im_eval extras, masked / observation-only launches, and the getup extras (PHC_FLAG_ZERO_OUT_FAR /
// PHC_FLAG_CYCLE_MOTION: env_im_x_getup_mcp.yaml) with the semantics documented at env_step.cu's GETUP variant.
//
// Deliberately the SIMPLE formulation: one warp per env, bodies strided over the lanes (j = lane, lane + 32), every record read
// straight from global memory through L1 / L2 and every output written straight to its row -- no shared-memory staging, no TMA.
// The arithmetic is phc_math.cuh, expression for expression as in env_step.cu.  These shapes are not the benchmarked
// configuration; the staged / specialised treatment of env_step.cu can follow once this path has run on hardware.
//
// STATUS: validated against the goldens of the unmodified reference (tests/golden/smplx.npz, g1.npz, and the 24-body goldens
// A-D) through the CPU emulation of this very source (tests/test_env_step_emu_cpu.py); it has not run on a GPU yet -- the
// GPU tests for it are opt-in (PHC_TEST_WIDE=1) until it has.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/phc_b200.h"
#include "phc_common.cuh"
#include "phc_math.cuh"

namespace phc {
namespace wide {

constexpr int kWarps = 4;
constexpr int kRec = 13;

struct Body { V3 p; Q4 q; V3 v; V3 w; };

__device__ __forceinline__ Body ld_body(const float* s) {
  Body b;
  b.p = v3(s[0], s[1], s[2]);
  b.q = q4(s[3], s[4], s[5], s[6]);
  b.v = v3(s[7], s[8], s[9]);
  b.w = v3(s[10], s[11], s[12]);
  return b;
}
// two-frame blend of one body: lerp pos(+offset)/vel/angvel, slerp rot (motion_lib_base.py:474-488)
__device__ __forceinline__ Body blend(const float* s0, const float* s1, float bl, V3 off) {
  const Body a = ld_body(s0), b = ld_body(s1);
  const float omb = 1.0f - bl;
  Body r;
  r.p = lerp3(a.p, b.p, omb, bl) + off;
  r.v = lerp3(a.v, b.v, omb, bl);
  r.w = lerp3(a.w, b.w, omb, bl);
  r.q = slerp(a.q, b.q, bl);
  return r;
}
__device__ __forceinline__ void put3(float* d, V3 v) { d[0] = v.x; d[1] = v.y; d[2] = v.z; }
__device__ __forceinline__ void put6(float* d, TanNorm t) { put3(d, t.t); put3(d + 3, t.n); }

// REC: the get-up schedule (PHC_FLAG_RECOVERY / PHC_FLAG_AMP_CURRENT, semantics at env_step.cu's REC variant); a template parameter so
// that the plain instantiation keeps its instruction stream.
template <bool REC = false>
__global__ void __launch_bounds__(kWarps * 32)
env_step_wide_kernel(const __grid_constant__ PhcStepArgs a, const int obs_dim, const int self_dim, const int amp_dim) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int env = blockIdx.x * kWarps + warp;
  if (env >= a.num_envs) return;                       // whole warp exits together
  if (a.only_where && a.only_where[env] == 0) return;  // masked subset (reset path)
  const uint32_t flags = a.flags;
  const bool obs_only = flags & PHC_FLAG_OBS_ONLY;
  const int J = a.lib.num_bodies, E = a.lib.num_ext_bodies;
  const bool robot = a.lib.num_dofs > 0;
  const int D = robot ? a.lib.num_dofs : 3 * (J - 1);
  const int T = a.time_steps;
  const int BS = a.lib.body_stride;
  const bool from_cache = (flags & PHC_FLAG_REWARD_FROM_CACHE) && !obs_only;

  const float* g_state = a.body_state + (size_t)env * a.bodies_per_env * kRec;
  const float* g_dof = a.dof_state + (size_t)env * D * 2;                  // (pos, vel) interleaved
  const int64_t progress = a.progress[env];
  // PHC_FLAG_RECOVERY (humanoid_im_getup.py:198-210): counter after the decrement; a recovering env keeps progress - 1 (observation too)
  int rcnt = 0;
  if (REC && (flags & PHC_FLAG_RECOVERY)) { const int c = a.recovery_counter[env]; rcnt = c - 1 < 0 ? 0 : c - 1; }
  const int64_t progress_o = (REC && rcnt > 0) ? progress - 1 : progress;
  const float t_start = a.start_times[env], t_off = a.start_offsets[env];
  const V3 goff = v3(a.global_offset[3 * env + 0], a.global_offset[3 * env + 1], a.global_offset[3 * env + 2]);
  float m_len, m_dt;
  int64_t m_nf, m_start;
  if (a.env_motion) {
    const PhcEnvMotion em = a.env_motion[env];
    m_len = em.len; m_dt = em.dt; m_nf = em.num_frames; m_start = em.start_row;
  } else {
    const int64_t mid = a.motion_ids[env];
    m_len = a.lib.motion_len[mid]; m_dt = a.lib.motion_dt[mid];
    m_nf = a.lib.motion_num_frames[mid]; m_start = a.lib.length_starts[mid];
  }
  const float* frames = a.lib.frames_body;
  float* const g_cache = a.ref_cache ? a.ref_cache + (size_t)env * BS : nullptr;

  // getup extras: motion parameters of the OBSERVATION time (re-based when the clip wraps this step, humanoid_im.py:1120-1146)
  const bool zof = flags & PHC_FLAG_ZERO_OUT_FAR;
  const bool cyc = (flags & PHC_FLAG_CYCLE_MOTION) && !obs_only;
  float t_start_o = t_start, t_off_o = t_off;
  V3 goff_o = goff;
  int cc = a.cycle_counter ? a.cycle_counter[env] : 0;
  bool rebased = false;
  if (cyc) {
    cc = cc - 1 < 0 ? 0 : cc - 1;                    // _update_cycle_count (humanoid_im.py:1076-1079)
    const float t_now0 = PHC_ADD(PHC_ADD(PHC_MUL((float)progress, a.dt), t_start), t_off);
    if (t_now0 >= m_len) {
      t_off_o = -PHC_MUL((float)progress, a.dt);
      const float grid = 1.0f / 30.0f;               // sample_time_interval (motion_lib_base.py:414-423)
      const long long k = (long long)((a.cycle_phase[env] * m_len) / grid);
      t_start_o = (float)k * grid;
      const Bracket32 b = frame_bracket32(t_start_o, m_len, (int)m_nf, m_dt);     // get_root_pos_smpl (:522-547)
      const float* r0 = frames + (size_t)(m_start + b.i0) * BS;
      const float* r1 = frames + (size_t)(m_start + b.i1) * BS;
      const float omb = 1.0f - b.blend;
      goff_o.x = g_state[0] - lerp1(r0[0], r1[0], omb, b.blend);
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
    __syncwarp();            // ... and the old counter before lane 0 stores the new one
    if (lane == 0 && a.cycle_counter) a.cycle_counter[env] = cc;
  }

  // heading frame of the simulated root
  const V3 root_p = v3(g_state[0], g_state[1], g_state[2]);
  Q4 root_q = q4(g_state[3], g_state[4], g_state[5], g_state[6]);
  if (!(flags & PHC_FLAG_UPRIGHT)) root_q = strip_base_rot(root_q);
  const float heading = heading_angle(root_q);
  const Q4 hq = quat_about_z(heading);
  const Q4 hinv = q4(0.0f, 0.0f, -hq.z, hq.w);
  const bool has_h = flags & PHC_FLAG_ROOT_HEIGHT_OBS;
  const int base0 = has_h ? 1 : 0;

  // ================= reward / reset at the CURRENT motion time (humanoid_im.py:879, :1118) ===========================
  // (the observation-only launch skips it, and writes the AMP vector below only with PHC_FLAG_AMP_CURRENT: the get-up reset path)
  const bool amp_cur = REC && obs_only && (flags & PHC_FLAG_AMP_CURRENT);
  if (!obs_only || amp_cur) {
   if (!obs_only) {
    const float t_now = PHC_ADD(PHC_ADD(PHC_MUL((float)progress, a.dt), t_start), t_off);
    Bracket32 br;
    br.i0 = 0; br.i1 = 0; br.blend = 0.f;
    if (!from_cache) br = frame_bracket32(t_now, m_len, (int)m_nf, m_dt);
    const float* f0 = frames + (size_t)(m_start + br.i0) * BS;
    const float* f1 = frames + (size_t)(m_start + br.i1) * BS;
    float e_pos = 0.f, e_rot = 0.f, e_vel = 0.f, e_ang = 0.f, mp = 0.f, cnt = 0.f, sum = 0.f, dist_root = 0.f;
    bool over = false;
    // a clip that wrapped this step: the reset test sees the pose at the re-based time (humanoid_im.py:1142, :1148)
    Bracket32 bt;
    bt.i0 = 0; bt.i1 = 0; bt.blend = 0.f;
    if (rebased) bt = frame_bracket32(PHC_ADD(PHC_ADD(PHC_MUL((float)progress, a.dt), t_start_o), t_off_o), m_len, (int)m_nf, m_dt);
    const float* q0 = frames + (size_t)(m_start + bt.i0) * BS;
    const float* q1 = frames + (size_t)(m_start + bt.i1) * BS;
    for (int jj = lane; jj < J + E; jj += 32) {
      const bool is_body = jj < J;
      Body sim;
      if (is_body) {
        sim = ld_body(g_state + jj * kRec);
      } else {       // extend body: parent_rot * pos_in_parent + parent_pos, rotation = the parent's (humanoid_im.py:917-919)
        sim = ld_body(g_state + a.ext_parent[jj - J] * kRec);
        sim.p = qrot(sim.q, v3(a.ext_pos[jj - J][0], a.ext_pos[jj - J][1], a.ext_pos[jj - J][2])) + sim.p;
      }
      const Body ref = from_cache ? ld_body(g_cache + jj * kRec) : blend(f0 + jj * kRec, f1 + jj * kRec, br.blend, goff);
      if (a.body_pos_gt && is_body) put3(a.body_pos_gt + ((size_t)env * J + jj) * 3, ref.p);
      const V3 dp = ref.p - sim.p;
      const float sp = dp.x * dp.x + dp.y * dp.y + dp.z * dp.z;
      e_pos += sp / 3.0f;
      const float ang = quat_angle(qmul(ref.q, qconj(sim.q)));
      e_rot += ang * ang;
      if (is_body) {
        const V3 dv = ref.v - sim.v, dw = ref.w - sim.w;
        e_vel += (dv.x * dv.x + dv.y * dv.y + dv.z * dv.z) / 3.0f;
        e_ang += (dw.x * dw.x + dw.y * dw.y + dw.z * dw.z) / 3.0f;
        const float dist = sqrtf(sp);
        mp += dist;
        if (jj == 0) dist_root = dist;
        float dist_t = dist;
        if (rebased) {
          const V3 pr = lerp3(v3(q0[jj * kRec], q0[jj * kRec + 1], q0[jj * kRec + 2]), v3(q1[jj * kRec], q1[jj * kRec + 1], q1[jj * kRec + 2]),
                              1.0f - bt.blend, bt.blend) + goff_o;
          const V3 d2 = pr - sim.p;
          dist_t = sqrtf(d2.x * d2.x + d2.y * d2.y + d2.z * d2.z);
        }
        const float thr = a.term_thresh[jj];
        if (thr < INFINITY) { cnt += 1.0f; sum += dist_t; }
        over = over || (dist_t > thr);
      }
    }
    if (a.mpjpe) {         // flags.im_eval extras (humanoid_im.py:674-680)
      const float m = warp_sum(mp) / (float)J;
      if (lane == 0) a.mpjpe[env] = m;
    }
    bool fallen;
    if (flags & PHC_FLAG_TERM_USE_MEAN) {
      const float c = warp_sum(cnt), s = warp_sum(sum);
      fallen = (s / c) > a.term_dist_mean;
    } else {
      fallen = __any_sync(0xffffffffu, over);
    }
    e_pos = warp_sum(e_pos) / (float)(J + E);
    e_rot = warp_sum(e_rot) / (float)(J + E);
    e_vel = warp_sum(e_vel) / (float)J;
    e_ang = warp_sum(e_ang) / (float)J;
    float power = 0.0f;
    if (a.dof_force) {
      const float* g_force = a.dof_force + (size_t)env * D;
      for (int d = lane; d < D; d += 32) power += fabsf(g_force[d] * g_dof[2 * d + 1]);
    }
    power = warp_sum(power);
    if (lane == 0) {
      const float r_pos = expf(-a.k_pos * e_pos), r_rot = expf(-a.k_rot * e_rot);
      const float r_vel = expf(-a.k_vel * e_vel), r_ang = expf(-a.k_ang_vel * e_ang);
      float rew = a.w_pos * r_pos + a.w_rot * r_rot + a.w_vel * r_vel + a.w_ang_vel * r_ang;
      const bool has_power = flags & PHC_FLAG_POWER_REWARD;
      float* raw = a.reward_raw + (size_t)env * (has_power ? 5 : 4);
      float w0 = r_pos, w1 = r_rot, w2 = r_vel, w3 = r_ang;
      if (zof) {            // point-goal mix (humanoid_im.py:890-905); lane 0 tracked the root
        const float pg = fminf(a.point_goal[env] - dist_root, 1.0f / 3.0f) * 9.0f;
        if (dist_root > 0.25f) { rew = pg; w0 = pg; w1 = 0.0f; w2 = 0.0f; w3 = 0.0f; }
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
      bool pass_time = t_now >= m_len;
      if (cyc) pass_time = progress >= (int64_t)a.max_episode_length - 1;      // pass_time_max (humanoid_im.py:1120-1124)
      int64_t terminated = 0;
      if (flags & PHC_FLAG_EARLY_TERM) {
        bool f = fallen && (progress > 1);
        if (flags & PHC_FLAG_NO_COLLISION) f = false;
        terminated = f ? 1 : 0;
      }
      int64_t reset = pass_time ? 1 : terminated;
      if (a.cycle_counter && !pass_time && cc > 0) { reset = 0; terminated = 0; }      // cc: this lane's own read (+ update)
      if (REC && rcnt > 0) { reset = 0; terminated = 0; }      // humanoid_im_getup.py:203-210: not cancelled by pass_time
      a.reset[env] = reset;
      a.terminate[env] = terminated;
    }
    if (REC && (flags & PHC_FLAG_RECOVERY)) {
      __syncwarp();          // every lane has read the counter and progress before lane 0 rewrites them
      if (lane == 0) {
        a.recovery_counter[env] = rcnt;
        if (rcnt > 0) const_cast<int64_t*>(a.progress)[env] = progress_o;
      }
    }
   }

    // ================= AMP observation of the simulated character -> slot 0 of its window ============================
    if (a.amp_out) {
      float* g_amp = a.amp_out + (size_t)env * a.amp_out_stride + (a.ring_head ? (size_t)(*a.ring_head) * (size_t)amp_dim : (size_t)0);
      if (a.amp_hist_in) {      // newest-first window shift, oldest slot first so that the in-place form is safe
        const float* h = a.amp_hist_in + (size_t)env * a.amp_out_stride;
        for (int s = a.amp_steps - 2; s >= 0; --s)
          for (int i = lane; i < amp_dim; i += 32) g_amp[(size_t)(s + 1) * amp_dim + i] = h[(size_t)s * amp_dim + i];
        __syncwarp();           // slot 0 is rewritten below by OTHER lanes than the ones that just copied it to slot 1
      }
      const int nj = a.num_amp_joints, nk = a.num_key_bodies;
      float* o = g_amp + base0;
      if (lane == 0) {
        const Body root = ld_body(g_state);
        if (has_h) g_amp[0] = root_p.z;
        put6(o, tan_norm((flags & PHC_FLAG_LOCAL_ROOT_OBS) ? qmul_zl(hinv, root_q) : root_q));
        put3(o + 6, qrot_z(hinv, root.v));
        put3(o + 9, qrot_z(hinv, root.w));
      }
      if (robot) {       // build_amp_observations_robot (humanoid_amp.py:1062-1104): raw hinge angles, then velocities
        for (int d = lane; d < D; d += 32) { o[12 + d] = g_dof[2 * d]; o[12 + D + d] = g_dof[2 * d + 1]; }
      } else {
        for (int k = lane; k < nj; k += 32) {
          const float* dj = g_dof + 6 * a.amp_joints[k];             // (pos, vel) pairs of the joint's 3 dofs
          put6(o + 12 + 6 * k, tan_norm(exp_map_to_quat(v3(dj[0], dj[2], dj[4]))));
          put3(o + 12 + 6 * nj + 3 * k, v3(dj[1], dj[3], dj[5]));
        }
      }
      if (lane < nk) {
        const float* kb = g_state + a.key_bodies[lane] * kRec;
        put3(o + 12 + (robot ? 2 * D : 9 * nj) + 3 * lane, qrot_z(hinv, v3(kb[0], kb[1], kb[2]) - root_p));
      }
    }
  }

  // ================= observation row: self obs + task obs v6 at the NEXT motion time(s) ================================
  float* const g_obs = a.obs + (size_t)env * a.obs_stride;
  if (lane == 0 && has_h) g_obs[0] = root_p.z;
  float* o_pos = g_obs + base0;
  float* o_rot = o_pos + 3 * (J - 1);
  float* o_vel = o_rot + 6 * J;
  float* o_ang = o_vel + 3 * J;
  for (int jj = lane; jj < J; jj += 32) {      // compute_humanoid_observations_smpl_max (humanoid.py:1994-2050)
    const Body sim = ld_body(g_state + jj * kRec);
    if (jj > 0) put3(o_pos + 3 * (jj - 1), qrot_z(hinv, sim.p - root_p));
    TanNorm tn = tan_norm(qmul_zl(hinv, sim.q));
    if (jj == 0 && !(flags & PHC_FLAG_LOCAL_ROOT_OBS)) tn = tan_norm(root_q);
    put6(o_rot + 6 * jj, tn);
    put3(o_vel + 3 * jj, qrot_z(hinv, sim.v));
    put3(o_ang + 3 * jj, qrot_z(hinv, sim.w));
  }
  for (int t = 0; t < T; ++t) {                // compute_imitation_observations_v6 (humanoid_im.py:1308-1358)
    float tn = PHC_MUL((float)(progress_o + 1), a.dt);
    if (T > 1) tn = PHC_ADD(tn, PHC_MUL((float)t, a.traj_dt));
    tn = PHC_ADD(PHC_ADD(tn, t_start_o), t_off_o);
    const Bracket32 b = frame_bracket32(tn, m_len, (int)m_nf, m_dt);
    const float* f0 = frames + (size_t)(m_start + b.i0) * BS;
    const float* f1 = frames + (size_t)(m_start + b.i1) * BS;
    float* tb = g_obs + self_dim + t * 24 * J;
    float dist_o = 0.0f;         // zero_out_far: |root_pos - reference root| at the observation time (humanoid_im.py:783-796)
    if (zof && t == 0) {
      const V3 rr = lerp3(v3(f0[0], f0[1], f0[2]), v3(f1[0], f1[1], f1[2]), 1.0f - b.blend, b.blend) + goff_o;
      const V3 dr = root_p - rr;
      dist_o = sqrtf(dr.x * dr.x + dr.y * dr.y + dr.z * dr.z);
      if (lane == 0) a.point_goal[env] = dist_o;
    }
    const int last = (t == 0 && g_cache) ? J + E : J;      // the pose cache also keeps the extend bodies of the first sample
    for (int jj = lane; jj < last; jj += 32) {
      const Body ref = blend(f0 + jj * kRec, f1 + jj * kRec, b.blend, goff_o);
      if (t == 0 && g_cache) {
        float* c = g_cache + jj * kRec;
        put3(c, ref.p); c[3] = ref.q.x; c[4] = ref.q.y; c[5] = ref.q.z; c[6] = ref.q.w; put3(c + 7, ref.v); put3(c + 10, ref.w);
      }
      if (jj >= J) continue;               // extend bodies: reward only, no observation columns
      const Body sim = ld_body(g_state + jj * kRec);
      Body ro = ref;               // what the observation sees as reference (cache / ref_* buffers keep `ref`)
      if (zof && t == 0) {
        if (dist_o > a.close_distance) {
          if (jj > 0) { ro.p = sim.p; ro.q = sim.q; }
          ro.v = sim.v; ro.w = sim.w;
        }
        if (dist_o > a.far_distance && jj == 0)
          ro.p = v3((ref.p.x - sim.p.x) / dist_o * a.far_distance + sim.p.x, (ref.p.y - sim.p.y) / dist_o * a.far_distance + sim.p.y,
                    (ref.p.z - sim.p.z) / dist_o * a.far_distance + sim.p.z);
      }
      put3(tb + 3 * jj, qrot_z(hinv, ro.p - sim.p));
      put6(tb + 3 * J + 6 * jj, tan_norm(qmul_zr(qmul_zl(hinv, qmul(ro.q, qconj(sim.q))), hq)));
      put3(tb + 9 * J + 3 * jj, qrot_z(hinv, ro.v - sim.v));
      put3(tb + 12 * J + 3 * jj, qrot_z(hinv, ro.w - sim.w));
      put3(tb + 15 * J + 3 * jj, qrot_z(hinv, ro.p - root_p));
      put6(tb + 18 * J + 6 * jj, tan_norm(qmul_zl(hinv, ro.q)));
      if (t == 0) {     // side buffers of _compute_task_obs(save_buffer=True)
        const size_t bj = (size_t)env * J + jj;
        if (a.ref_body_pos) put3(a.ref_body_pos + 3 * bj, ref.p);
        if (a.ref_body_vel) put3(a.ref_body_vel + 3 * bj, ref.v);
        if (a.ref_body_ang_vel) put3(a.ref_body_ang_vel + 3 * bj, ref.w);
        if (a.ref_body_rot) { float* d = a.ref_body_rot + 4 * bj; d[0] = ref.q.x; d[1] = ref.q.y; d[2] = ref.q.z; d[3] = ref.q.w; }
      }
    }
  }
}

}  // namespace wide
}  // namespace phc

extern "C" void phc_set_error(const char* msg);
extern "C" int phc_check_cuda(cudaError_t e, const char* what);
extern "C" void phc_count_launches(int n);

// called by phc_env_step (env_step.cu) after its argument validation, when J + E > PHC_LANE_BODIES
extern "C" int phc_env_step_wide_launch(const PhcStepArgs* a, int obs_dim, int self_dim, int amp_dim, void* stream) {
  using namespace phc::wide;
  const int grid = (a->num_envs + kWarps - 1) / kWarps;
  if (a->flags & (PHC_FLAG_RECOVERY | PHC_FLAG_AMP_CURRENT))
    env_step_wide_kernel<true><<<grid, kWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(*a, obs_dim, self_dim, amp_dim);
  else
    env_step_wide_kernel<<<grid, kWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(*a, obs_dim, self_dim, amp_dim);
  phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "env_step_wide_kernel launch");
}
