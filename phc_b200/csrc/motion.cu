// Motion-library kernels: table packing, the general get_motion_state query and the AMP "demo" observation of
// the reference motion.  Reference: phc/utils/motion_lib_base.py:300-307 (tables), :437-520 (get_motion_state),
// :549-567 (_calc_frame_blend, _local_rotation_to_dof_smpl); phc/env/tasks/humanoid_amp.py:253-284, :575-603, :966-1011.
//
// These are the off-step paths (episode resets, discriminator demo batches): one warp per query, lane = body,
// plain cached loads of the packed records (a frame bracket is 2 x 1.2 KB contiguous).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/phc_b200.h"
#include "phc_common.cuh"
#include "phc_math.cuh"
#include "motion_sample.cuh"

extern "C" void phc_set_error(const char* msg);
extern "C" int phc_check_cuda(cudaError_t e, const char* what);
extern "C" void phc_count_launches(int n);

namespace phc {

__global__ void motion_pack_kernel(const float* __restrict__ gts, const float* __restrict__ grs,
                                   const float* __restrict__ gvs, const float* __restrict__ gavs,
                                   const float* __restrict__ lrs, const float* __restrict__ dvs, int64_t F, int J,
                                   int BS, int JS, float* __restrict__ fb, float* __restrict__ fj) {
  const int64_t total = F * J;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = i / J;
    const int j = (int)(i - f * J);
    float* o = fb + f * BS + j * kRec;
    const float* p = gts + i * 3;
    const float* q = grs + i * 4;
    const float* v = gvs + i * 3;
    const float* w = gavs + i * 3;
    o[0] = p[0]; o[1] = p[1]; o[2] = p[2];
    o[3] = q[0]; o[4] = q[1]; o[5] = q[2]; o[6] = q[3];
    o[7] = v[0]; o[8] = v[1]; o[9] = v[2];
    o[10] = w[0]; o[11] = w[1]; o[12] = w[2];
    if (j == 0) for (int k = J * kRec; k < BS; ++k) fb[f * BS + k] = 0.0f;
    if (fj) {
      float* oj = fj + f * JS;
      const float* lq = lrs + i * 4;
      oj[4 * j + 0] = lq[0]; oj[4 * j + 1] = lq[1]; oj[4 * j + 2] = lq[2]; oj[4 * j + 3] = lq[3];
      if (j > 0) {
        const float* dv = dvs + (f * (J - 1) + (j - 1)) * 3;
        float* od = oj + 4 * J + 3 * (j - 1);
        od[0] = dv[0]; od[1] = dv[1]; od[2] = dv[2];
      } else {
        for (int k = 4 * J + 3 * (J - 1); k < JS; ++k) oj[k] = 0.0f;
      }
    }
  }
}

__global__ void motion_pack_dofs_kernel(const float* __restrict__ dof_pos, const float* __restrict__ dof_vel, int64_t F, int D, int JS,
                                        float* __restrict__ fj) {
  const int64_t total = F * JS;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = i / JS;
    const int c = (int)(i - f * JS);
    fj[i] = c < D ? dof_pos[f * D + c] : (c < 2 * D ? dof_vel[f * D + (c - D)] : 0.0f);
  }
}

__global__ void __launch_bounds__(128)
motion_state_kernel(const __grid_constant__ PhcMotionLib lib, const int64_t* __restrict__ ids,
                    const float* __restrict__ times, const float* __restrict__ offset, int64_t n,
                    const __grid_constant__ PhcMotionStateOut out) {
  const int64_t qi = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (qi >= n) return;
  const int J = lib.num_bodies, JE = J + lib.num_ext_bodies, D = lib.num_dofs;
  if (lane >= JE && lane >= D) return;
  const V3 off = offset ? v3(offset[3 * qi], offset[3 * qi + 1], offset[3 * qi + 2]) : v3(0.f, 0.f, 0.f);
  const bool want_joint = (out.dof_pos != nullptr) || (out.dof_vel != nullptr);
  MotionSample s = sample_motion(lib, ids[qi], times[qi], v3(0.f, 0.f, 0.f), lane, want_joint);
  if (offset) s.body.p = s.body.p + off;          // the reference adds the offset only when one is given
  if (lane < JE) {                                 // robots: all J + E bodies (the *_t outputs)
    const int64_t bt = qi * JE + lane;
    if (out.rg_pos_t) st3g(out.rg_pos_t + 3 * bt, s.body.p);
    if (out.rg_rot_t) st4g(out.rg_rot_t + 4 * bt, s.body.q);
    if (out.body_vel_t) st3g(out.body_vel_t + 3 * bt, s.body.v);
    if (out.body_ang_vel_t) st3g(out.body_ang_vel_t + 3 * bt, s.body.w);
  }
  if (lane < J) {
    const int64_t bj = qi * J + lane;
    if (out.rg_pos) st3g(out.rg_pos + 3 * bj, s.body.p);
    if (out.rb_rot) st4g(out.rb_rot + 4 * bj, s.body.q);
    if (out.body_vel) st3g(out.body_vel + 3 * bj, s.body.v);
    if (out.body_ang_vel) st3g(out.body_ang_vel + 3 * bj, s.body.w);
  }
  if (D > 0) {
    if (lane < D) {
      if (out.dof_pos) out.dof_pos[qi * D + lane] = s.dof_pos.x;
      if (out.dof_vel) out.dof_vel[qi * D + lane] = s.dof_vel.x;
    }
  } else if (lane > 0 && lane < J) {
    const int64_t dj = qi * (J - 1) + (lane - 1);
    if (out.dof_pos) st3g(out.dof_pos + 3 * dj, s.dof_pos);
    if (out.dof_vel) st3g(out.dof_vel + 3 * dj, s.dof_vel);
  }
  if (lane == 0) {
    if (out.root_pos) st3g(out.root_pos + 3 * qi, s.body.p);
    if (out.root_rot) st4g(out.root_rot + 4 * qi, s.body.q);
    if (out.root_vel) st3g(out.root_vel + 3 * qi, s.body.v);
    if (out.root_ang_vel) st3g(out.root_ang_vel + 3 * qi, s.body.w);
  }
}

struct AmpDemoArgs {
  PhcMotionLib lib;
  const int64_t* ids;
  const float* times0;
  int64_t n;
  int32_t first_step, num_steps;
  float dt;
  uint32_t flags;
  int32_t key_bodies[PHC_MAX_KEY_BODIES];
  int32_t num_key_bodies;
  int32_t amp_joints[PHC_MAX_AMP_JOINTS];
  int32_t num_amp_joints;
  float* out;
  int64_t out_stride;
  const int64_t* only_where;
  int32_t slot_offset;      // ring rotation: logical step k is written to physical slot (k + slot_offset) % num_steps
  const int32_t* slot_offset_dev;   // optional: the rotation read from device memory (the ring head HumanoidIm keeps on the device)
};

// warp per (sample, history step): motion sample at t0 - (first_step + k) dt, then build_amp_observations_smpl
__global__ void __launch_bounds__(128) amp_demo_kernel(const __grid_constant__ AmpDemoArgs a) {
  const int64_t wi = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (wi >= a.n * a.num_steps) return;
  const int64_t si = wi / a.num_steps;
  if (a.only_where && a.only_where[si] == 0) return;
  const int k = (int)(wi - si * a.num_steps);
  const int J = a.lib.num_bodies;
  // motion_times0 + (-dt * (k + first)) : humanoid_amp.py:257-261 / :577-582
  const float t = a.times0[si] + (-a.dt * (float)(k + a.first_step));
  const int D = a.lib.num_dofs;
  const int j = (lane < J || lane < D) ? lane : 0;
  const MotionSample s = sample_motion(a.lib, a.ids[si], t, v3(0.f, 0.f, 0.f), j, true);
  // root record broadcast from lane 0
  BodyS r;
  r.p = v3(__shfl_sync(0xffffffffu, s.body.p.x, 0), __shfl_sync(0xffffffffu, s.body.p.y, 0), __shfl_sync(0xffffffffu, s.body.p.z, 0));
  r.q = q4(__shfl_sync(0xffffffffu, s.body.q.x, 0), __shfl_sync(0xffffffffu, s.body.q.y, 0), __shfl_sync(0xffffffffu, s.body.q.z, 0), __shfl_sync(0xffffffffu, s.body.q.w, 0));
  r.v = v3(__shfl_sync(0xffffffffu, s.body.v.x, 0), __shfl_sync(0xffffffffu, s.body.v.y, 0), __shfl_sync(0xffffffffu, s.body.v.z, 0));
  r.w = v3(__shfl_sync(0xffffffffu, s.body.w.x, 0), __shfl_sync(0xffffffffu, s.body.w.y, 0), __shfl_sync(0xffffffffu, s.body.w.z, 0));
  if (lane >= J && lane >= D) return;

  const bool upright = a.flags & PHC_FLAG_UPRIGHT, has_h = a.flags & PHC_FLAG_ROOT_HEIGHT_OBS;
  const Q4 root_q = upright ? r.q : strip_base_rot(r.q);
  const Q4 hinv = quat_about_z(-heading_angle(root_q));
  const int nj = a.num_amp_joints, nk = a.num_key_bodies;
  const int kp = (k + (a.slot_offset_dev ? *a.slot_offset_dev : a.slot_offset)) % a.num_steps;
  const int row = has_h + 12 + (D > 0 ? 2 * D : 9 * nj) + 3 * nk;
  float* o = a.out + si * a.out_stride + (int64_t)kp * row + (has_h ? 1 : 0);
  if (D > 0) {       // build_amp_observations_robot (humanoid_amp.py:1062-1104): raw hinge angles and velocities
    if (lane == 0) {
      if (has_h) o[-1] = r.p.z;
      const TanNorm tn = tan_norm((a.flags & PHC_FLAG_LOCAL_ROOT_OBS) ? qmul(hinv, root_q) : root_q);
      st3g(o, tn.t); st3g(o + 3, tn.n);
      st3g(o + 6, qrot_z(hinv, r.v));
      st3g(o + 9, qrot_z(hinv, r.w));
    }
    if (lane < D) { o[12 + lane] = s.dof_pos.x; o[12 + D + lane] = s.dof_vel.x; }
    if (lane < J)
      for (int kk = 0; kk < nk; ++kk)
        if (a.key_bodies[kk] == lane) st3g(o + 12 + 2 * D + 3 * kk, qrot_z(hinv, s.body.p - r.p));
    return;
  }
  if (lane == 0) {
    if (has_h) o[-1] = r.p.z;
    const TanNorm tn = tan_norm((a.flags & PHC_FLAG_LOCAL_ROOT_OBS) ? qmul(hinv, root_q) : root_q);
    st3g(o, tn.t); st3g(o + 3, tn.n);
    st3g(o + 6, qrot_z(hinv, r.v));
    st3g(o + 9, qrot_z(hinv, r.w));
  } else {
    for (int kk = 0; kk < nj; ++kk)
      if (a.amp_joints[kk] == lane - 1) {
        const TanNorm tn = tan_norm(exp_map_to_quat(s.dof_pos));
        st3g(o + 12 + 6 * kk, tn.t); st3g(o + 12 + 6 * kk + 3, tn.n);
        st3g(o + 12 + 6 * nj + 3 * kk, s.dof_vel);
      }
  }
  for (int kk = 0; kk < nk; ++kk)
    if (a.key_bodies[kk] == lane) st3g(o + 12 + 9 * nj + 3 * kk, qrot_z(hinv, s.body.p - r.p));
}

__global__ void env_motion_gather_kernel(const __grid_constant__ PhcMotionLib lib, const int64_t* __restrict__ ids, int64_t n,
                                         PhcEnvMotion* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t m = ids[i];
  PhcEnvMotion e;
  e.len = lib.motion_len[m]; e.dt = lib.motion_dt[m];
  e.num_frames = (int32_t)lib.motion_num_frames[m]; e.start_row = (int32_t)lib.length_starts[m];
  out[i] = e;
}

// Reset bookkeeping of the selected envs in one pass (Humanoid._reset_envs / HumanoidIm._reset_task, humanoid_im.py:955-1023):
// new start time on the 1/30 s grid from a uniform phase (MotionLibBase.sample_time_interval, motion_lib_base.py:414-423),
// start offset / global offset / cycle counter / progress / reset / terminate cleared.
__global__ void reset_bookkeeping_kernel(const int64_t* __restrict__ mask, const float* __restrict__ phase,
                                         const PhcEnvMotion* __restrict__ em, int64_t n, float* __restrict__ start_times,
                                         float* __restrict__ start_offsets, float* __restrict__ global_offset,
                                         int32_t* __restrict__ cycle_counter, int64_t* __restrict__ progress,
                                         int64_t* __restrict__ reset, int64_t* __restrict__ terminate) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || mask[i] == 0) return;
  const float grid = 1.0f / 30.0f;
  const long long k = (long long)((phase[i] * em[i].len) / grid);          // .long(): truncation
  start_times[i] = (float)k * grid;
  start_offsets[i] = 0.0f;
  global_offset[3 * i] = 0.0f; global_offset[3 * i + 1] = 0.0f; global_offset[3 * i + 2] = 0.0f;
  if (cycle_counter) cycle_counter[i] = 0;
  progress[i] = 0;
  if (reset) reset[i] = 0;
  if (terminate) terminate[i] = 0;
}

// Reset path: write the reference pose at (id, time) of every env with mask != 0 into the simulator tensors
// (HumanoidAMP._set_env_state, humanoid_amp.py:605-637: rigid-body rows + dof pos/vel), warp per env.
__global__ void __launch_bounds__(128)
set_env_state_kernel(const __grid_constant__ PhcMotionLib lib, const int64_t* __restrict__ ids,
                     const float* __restrict__ times, const float* __restrict__ offset,
                     const int64_t* __restrict__ only_where, int64_t n, float* __restrict__ body_state, int bpe,
                     float* __restrict__ dof_state) {
  const int64_t env = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (env >= n) return;
  if (only_where && only_where[env] == 0) return;
  const int J = lib.num_bodies, D = lib.num_dofs;
  if (lane >= J && lane >= D) return;
  const V3 off = offset ? v3(offset[3 * env], offset[3 * env + 1], offset[3 * env + 2]) : v3(0.f, 0.f, 0.f);
  MotionSample s = sample_motion(lib, ids[env], times[env], v3(0.f, 0.f, 0.f), lane, dof_state != nullptr);
  if (offset) s.body.p = s.body.p + off;
  if (D > 0 && dof_state && lane < D) {                       // hinge joints: [D, 2] (pos, vel)
    float* d = dof_state + ((size_t)env * D + lane) * 2;
    d[0] = s.dof_pos.x; d[1] = s.dof_vel.x;
  }
  if (lane >= J) return;
  float* o = body_state + ((size_t)env * bpe + lane) * kRec;
  o[0] = s.body.p.x; o[1] = s.body.p.y; o[2] = s.body.p.z;
  o[3] = s.body.q.x; o[4] = s.body.q.y; o[5] = s.body.q.z; o[6] = s.body.q.w;
  o[7] = s.body.v.x; o[8] = s.body.v.y; o[9] = s.body.v.z;
  o[10] = s.body.w.x; o[11] = s.body.w.y; o[12] = s.body.w.z;
  if (D == 0 && dof_state && lane > 0) {
    float* d = dof_state + ((size_t)env * (J - 1) + (lane - 1)) * 6;      // [D, 2] interleaved (pos, vel)
    d[0] = s.dof_pos.x; d[1] = s.dof_vel.x; d[2] = s.dof_pos.y; d[3] = s.dof_vel.y; d[4] = s.dof_pos.z; d[5] = s.dof_vel.z;
  }
}

// AMP ring -> newest-first window: out[n, k, :] = ring[n, (head + k) % S, :]   (pure copy, float4 when A % 4 == 0)
__global__ void amp_window_export_kernel(const float* __restrict__ ring, int64_t ring_stride, int64_t n, int S, int A, int head_arg,
                                         const int32_t* __restrict__ head_dev, float* __restrict__ out, int64_t out_stride) {
  const int head = head_dev ? *head_dev : head_arg;
  if ((A & 3) == 0 && (ring_stride & 3) == 0 && (out_stride & 3) == 0) {
    const int A4 = A >> 2;
    const int64_t total = n * S * A4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
      const int64_t e = i / (S * A4);
      const int r = (int)(i - e * S * A4);
      const int k = r / A4, c = r - k * A4;
      const int kp = (head + k) % S;
      reinterpret_cast<float4*>(out + e * out_stride)[k * A4 + c] = reinterpret_cast<const float4*>(ring + e * ring_stride)[kp * A4 + c];
    }
  } else {
    const int64_t total = n * S * A;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
      const int64_t e = i / (S * A);
      const int r = (int)(i - e * S * A);
      const int k = r / A, c = r - k * A;
      out[e * out_stride + k * A + c] = ring[e * ring_stride + ((head + k) % S) * A + c];
    }
  }
}

}  // namespace phc

extern "C" int phc_motion_body_stride(int32_t J) { return (13 * J + 3) & ~3; }
extern "C" int phc_motion_joint_stride(int32_t J) { return (4 * J + 3 * (J - 1) + 3) & ~3; }
extern "C" int phc_motion_dof_stride(int32_t D) { return (2 * D + 3) & ~3; }

extern "C" int phc_motion_pack_dofs(const float* dof_pos, const float* dof_vel, int64_t F, int32_t D, float* fj, void* stream) {
  if (!dof_pos || !dof_vel || !fj || F < 0 || D < 1 || (reinterpret_cast<uintptr_t>(fj) & 15)) { phc_set_error("phc_motion_pack_dofs: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (F == 0) return PHC_OK;
  const int JS = phc_motion_dof_stride(D);
  int64_t g = (F * JS + 255) / 256; if (g > 132 * 16) g = 132 * 16;
  phc::motion_pack_dofs_kernel<<<(unsigned)g, 256, 0, static_cast<cudaStream_t>(stream)>>>(dof_pos, dof_vel, F, D, JS, fj); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "motion_pack_dofs_kernel launch");
}

extern "C" int phc_motion_pack(const float* gts, const float* grs, const float* gvs, const float* gavs,
                               const float* lrs, const float* dvs, int64_t F, int32_t J, float* fb, float* fj,
                               void* stream) {
  if (!gts || !grs || !gvs || !gavs || !fb || F < 0 || J < 1) { phc_set_error("phc_motion_pack: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if ((reinterpret_cast<uintptr_t>(fb) & 15) || (fj && (reinterpret_cast<uintptr_t>(fj) & 15))) {
    phc_set_error("phc_motion_pack: packed tables must be 16-byte aligned"); return PHC_ERR_INVALID_ARG;
  }
  if (F == 0) return PHC_OK;
  const bool joint = fj && lrs && dvs;
  const int64_t total = F * J;
  const int block = 256;
  const int grid = (int)((total + block - 1) / block < 132 * 16 ? (total + block - 1) / block : 132 * 16);
  phc::motion_pack_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(
      gts, grs, gvs, gavs, lrs, dvs, F, J, phc_motion_body_stride(J), phc_motion_joint_stride(J), fb, joint ? fj : nullptr); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "motion_pack_kernel launch");
}

static int check_lib(const PhcMotionLib* lib, const char* who) {
  if (!lib || !lib->frames_body || !lib->motion_len || !lib->motion_dt || !lib->motion_num_frames || !lib->length_starts) {
    phc_set_error("motion library has NULL tables"); return PHC_ERR_INVALID_ARG;
  }
  if (lib->num_bodies < 1 || lib->num_ext_bodies < 0 || lib->num_ext_bodies > PHC_MAX_EXT_BODIES || lib->num_dofs < 0 ||
      lib->body_stride != phc_motion_body_stride(lib->num_bodies + lib->num_ext_bodies) ||
      (lib->frames_joint && lib->joint_stride != (lib->num_dofs > 0 ? phc_motion_dof_stride(lib->num_dofs)
                                                                     : phc_motion_joint_stride(lib->num_bodies)))) {
    phc_set_error("motion library strides do not match num_bodies / num_ext_bodies / num_dofs (use phc_motion_pack[_dofs])"); return PHC_ERR_INVALID_ARG;
  }
  if (lib->num_bodies + lib->num_ext_bodies > PHC_MAX_BODIES || lib->num_dofs > 2 * PHC_MAX_BODIES) {
    phc_set_error("more than PHC_MAX_BODIES bodies (incl. extend bodies) or 2 * PHC_MAX_BODIES hinge dofs"); return PHC_ERR_UNSUPPORTED;
  }
  (void)who;
  return PHC_OK;
}
// more than one body (or hinge dof) per lane: the strided kernels of motion_wide.cu
static bool is_wide(const PhcMotionLib* lib) { return lib->num_bodies + lib->num_ext_bodies > PHC_LANE_BODIES || lib->num_dofs > PHC_LANE_BODIES; }
extern "C" int phc_motion_state_wide_launch(const PhcMotionLib* lib, const int64_t* ids, const float* times, const float* offset,
                                            int64_t n, const PhcMotionStateOut* out, void* stream);
extern "C" int phc_amp_obs_demo_wide_launch(const PhcMotionLib* lib, const int64_t* ids, const float* times0, int64_t n, int32_t first_step,
                                            int32_t num_steps, float dt, uint32_t flags, const int32_t* key_bodies, int32_t nk,
                                            const int32_t* amp_joints, int32_t nj, float* out, int64_t out_stride,
                                            const int64_t* only_where, int32_t slot_offset, const int32_t* slot_offset_dev, void* stream);
extern "C" int phc_set_env_state_wide_launch(const PhcMotionLib* lib, const int64_t* ids, const float* times, const float* offset,
                                             const int64_t* only_where, int64_t n, float* body_state, int32_t bodies_per_env,
                                             float* dof_state, void* stream);

extern "C" int phc_motion_state(const PhcMotionLib* lib, const int64_t* ids, const float* times, const float* offset,
                                int64_t n, const PhcMotionStateOut* out, void* stream) {
  int rc = check_lib(lib, "phc_motion_state");
  if (rc) return rc;
  if (!ids || !times || !out || n < 0) { phc_set_error("phc_motion_state: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if ((out->dof_pos || out->dof_vel) && !lib->frames_joint) { phc_set_error("phc_motion_state: dof outputs need frames_joint"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  if (is_wide(lib)) return phc_motion_state_wide_launch(lib, ids, times, offset, n, out, stream);
  const int wpb = 4;
  const int64_t grid = (n + wpb - 1) / wpb;
  phc::motion_state_kernel<<<(unsigned)grid, wpb * 32, 0, static_cast<cudaStream_t>(stream)>>>(*lib, ids, times, offset, n, *out); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "motion_state_kernel launch");
}

extern "C" int phc_amp_obs_demo(const PhcMotionLib* lib, const int64_t* ids, const float* times0, int64_t n,
                                int32_t first_step, int32_t num_steps, float dt, uint32_t flags,
                                const int32_t* key_bodies, int32_t nk, const int32_t* amp_joints, int32_t nj, float* out,
                                int64_t out_stride, const int64_t* only_where, int32_t slot_offset, void* stream) {
  return phc_amp_obs_demo_ring(lib, ids, times0, n, first_step, num_steps, dt, flags, key_bodies, nk, amp_joints, nj, out, out_stride, only_where,
                               slot_offset, nullptr, stream);
}

extern "C" int phc_amp_obs_demo_ring(const PhcMotionLib* lib, const int64_t* ids, const float* times0, int64_t n,
                                     int32_t first_step, int32_t num_steps, float dt, uint32_t flags,
                                     const int32_t* key_bodies, int32_t nk, const int32_t* amp_joints, int32_t nj, float* out,
                                     int64_t out_stride, const int64_t* only_where, int32_t slot_offset, const int32_t* slot_offset_dev,
                                     void* stream) {
  int rc = check_lib(lib, "phc_amp_obs_demo");
  if (rc) return rc;
  if (!lib->frames_joint) { phc_set_error("phc_amp_obs_demo: needs frames_joint"); return PHC_ERR_INVALID_ARG; }
  if (!ids || !times0 || !out || n < 0 || num_steps < 1 || nk < 0 || nk > PHC_MAX_KEY_BODIES || nj < 0 || nj > PHC_MAX_AMP_JOINTS || (nj > 0 && !amp_joints) || (nk > 0 && !key_bodies)) {
    phc_set_error("phc_amp_obs_demo: bad arguments"); return PHC_ERR_INVALID_ARG;
  }
  const int A = lib->num_dofs > 0 ? phc_amp_obs_dim_robot(lib->num_dofs, nk, flags) : phc_amp_obs_dim(nj, nk, flags);
  if (out_stride < (int64_t)num_steps * A) { phc_set_error("phc_amp_obs_demo: out_stride too small"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  if (is_wide(lib)) return phc_amp_obs_demo_wide_launch(lib, ids, times0, n, first_step, num_steps, dt, flags, key_bodies, nk, amp_joints, nj, out,
                                                         out_stride, only_where, slot_offset, slot_offset_dev, stream);
  phc::AmpDemoArgs a;
  a.lib = *lib; a.ids = ids; a.times0 = times0; a.n = n; a.first_step = first_step; a.num_steps = num_steps; a.dt = dt;
  a.flags = flags; a.num_key_bodies = nk; a.num_amp_joints = nj;
  for (int i = 0; i < PHC_MAX_AMP_JOINTS; ++i) a.amp_joints[i] = i < nj ? amp_joints[i] : -1; a.out = out; a.out_stride = out_stride; a.only_where = only_where;
  a.slot_offset = ((slot_offset % num_steps) + num_steps) % num_steps;
  a.slot_offset_dev = slot_offset_dev;
  for (int i = 0; i < PHC_MAX_KEY_BODIES; ++i) a.key_bodies[i] = i < nk ? key_bodies[i] : -1;
  const int wpb = 4;
  const int64_t warps = n * num_steps;
  phc::amp_demo_kernel<<<(unsigned)((warps + wpb - 1) / wpb), wpb * 32, 0, static_cast<cudaStream_t>(stream)>>>(a); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "amp_demo_kernel launch");
}

extern "C" int phc_set_env_state(const PhcMotionLib* lib, const int64_t* ids, const float* times, const float* offset,
                                 const int64_t* only_where, int64_t n, float* body_state, int32_t bodies_per_env,
                                 float* dof_state, void* stream) {
  int rc = check_lib(lib, "phc_set_env_state");
  if (rc) return rc;
  if (!ids || !times || !body_state || n < 0 || bodies_per_env < lib->num_bodies) { phc_set_error("phc_set_env_state: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (dof_state && !lib->frames_joint) { phc_set_error("phc_set_env_state: dof_state needs frames_joint"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  if (is_wide(lib)) return phc_set_env_state_wide_launch(lib, ids, times, offset, only_where, n, body_state, bodies_per_env, dof_state, stream);
  const int wpb = 4;
  phc::set_env_state_kernel<<<(unsigned)((n + wpb - 1) / wpb), wpb * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      *lib, ids, times, offset, only_where, n, body_state, bodies_per_env, dof_state); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "set_env_state_kernel launch");
}

extern "C" int phc_amp_window_export(const float* ring, int64_t ring_stride, int64_t n, int32_t num_steps, int32_t amp_dim,
                                     int32_t head, float* out, int64_t out_stride, void* stream) {
  return phc_amp_window_export_ring(ring, ring_stride, n, num_steps, amp_dim, head, nullptr, out, out_stride, stream);
}

namespace phc {
__global__ void ring_advance_kernel(int32_t* head, int32_t slots) { *head = (*head - 1 + slots) % slots; }
}  // namespace phc

extern "C" int phc_ring_advance(int32_t* head, int32_t num_slots, void* stream) {
  if (!head || num_slots < 1) { phc_set_error("phc_ring_advance: bad arguments"); return PHC_ERR_INVALID_ARG; }
  phc::ring_advance_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(head, num_slots); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "ring_advance_kernel launch");
}

extern "C" int phc_amp_window_export_ring(const float* ring, int64_t ring_stride, int64_t n, int32_t num_steps, int32_t amp_dim,
                                          int32_t head, const int32_t* head_dev, float* out, int64_t out_stride, void* stream) {
  if (!ring || !out || n < 0 || num_steps < 1 || amp_dim < 1 || head < 0 || head >= num_steps ||
      ring_stride < (int64_t)num_steps * amp_dim || out_stride < (int64_t)num_steps * amp_dim) {
    phc_set_error("phc_amp_window_export: bad arguments"); return PHC_ERR_INVALID_ARG;
  }
  if (n == 0) return PHC_OK;
  if ((reinterpret_cast<uintptr_t>(ring) | reinterpret_cast<uintptr_t>(out)) & 15) { phc_set_error("phc_amp_window_export: buffers must be 16-byte aligned"); return PHC_ERR_INVALID_ARG; }
  int64_t g = (n * num_steps * amp_dim / 4 + 255) / 256; if (g > 132 * 16) g = 132 * 16; if (g < 1) g = 1;
  phc::amp_window_export_kernel<<<(unsigned)g, 256, 0, static_cast<cudaStream_t>(stream)>>>(ring, ring_stride, n, num_steps, amp_dim, head, head_dev, out, out_stride); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "amp_window_export_kernel launch");
}

extern "C" int phc_env_motion_gather(const PhcMotionLib* lib, const int64_t* ids, int64_t n, PhcEnvMotion* out, void* stream) {
  int rc = check_lib(lib, "phc_env_motion_gather");
  if (rc) return rc;
  if (!ids || !out || n < 0 || (reinterpret_cast<uintptr_t>(out) & 15)) { phc_set_error("phc_env_motion_gather: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (lib->num_frames_total >= (int64_t)1 << 31) { phc_set_error("phc_env_motion_gather: frame table too large for 32-bit rows"); return PHC_ERR_UNSUPPORTED; }
  if (n == 0) return PHC_OK;
  phc::env_motion_gather_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(*lib, ids, n, out); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "env_motion_gather_kernel launch");
}

extern "C" int phc_reset_bookkeeping(const int64_t* mask, const float* phase, const PhcEnvMotion* env_motion, int64_t n,
                                     float* start_times, float* start_offsets, float* global_offset, int32_t* cycle_counter,
                                     int64_t* progress, int64_t* reset, int64_t* terminate, void* stream) {
  if (n == 0) return PHC_OK;
  if (!mask || !phase || !env_motion || n < 0 || !start_times || !start_offsets || !global_offset || !progress) {
    phc_set_error("phc_reset_bookkeeping: bad arguments"); return PHC_ERR_INVALID_ARG;
  }
  phc::reset_bookkeeping_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      mask, phase, env_motion, n, start_times, start_offsets, global_offset, cycle_counter, progress, reset, terminate); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "reset_bookkeeping_kernel launch");
}
