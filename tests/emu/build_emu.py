"""TEST INFRASTRUCTURE: assemble and compile the CPU emulation of the fused env-step kernel FROM THE PRODUCT SOURCES.

The translation unit is: the emulation prelude (tests/emu/cuda_emu_prelude.h, phc_common_emu.cuh) + `warp_sum` / `warp_sum4`
cut verbatim out of phc_b200/csrc/phc_common.cuh + include/phc_b200.h + phc_b200/csrc/phc_math.cuh + the `namespace phc { ... }`
part of phc_b200/csrc/env_step.cu (layout helpers and `env_step_kernel`, verbatim) + the same part of env_step_wide.cu (the strided kernel for more than 32 bodies)
+ a launcher that runs one warp (32 std::threads) per env.  Nothing of the kernel is restated here."""
import os
import re
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "phc_b200", "csrc")

LAUNCHER = r'''
namespace phc { alignas(128) float smem[1 << 16]; }      // the kernel's `extern __shared__ float smem[]`
namespace phc { namespace fast { alignas(128) float smem[1 << 16]; } }

template <int T_MAX, int JT, bool GETUP, bool FAST>
static void emu_launch(const PhcStepArgs& a, int obs_dim, int self_dim, int amp_dim, bool alias_obs, bool state_bulk_ok) {
  for (int env = 0; env < a.num_envs; ++env) {
    EmuWarp warp;
    std::vector<std::thread> lanes;
    for (int lane = 0; lane < 32; ++lane)
      lanes.emplace_back([&, lane] {
        emu_warp = &warp;
        emu_lane = lane;
        threadIdx.x = (unsigned)((env % phc::kWarpsPerCta) * 32 + lane); threadIdx.y = threadIdx.z = 0;
        blockIdx.x = (unsigned)(env / phc::kWarpsPerCta); blockIdx.y = blockIdx.z = 0;
        phc::env_step_kernel<T_MAX, JT, GETUP, FAST>(a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok);
      });
    for (auto& t : lanes) t.join();
  }
}

extern "C" int emu_env_step(const PhcStepArgs* a, int obs_dim, int self_dim, int amp_dim, int alias_obs, int state_bulk_ok, int variant) {
  switch (variant) {
    case 0: emu_launch<1, 24, false, false>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 1: emu_launch<1, 24, false, true>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 2: emu_launch<1, 24, true, false>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 3: emu_launch<1, 0, false, false>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 4: emu_launch<4, 0, false, false>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 5: emu_launch<1, 0, true, false>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 7: {    // env_step_fast.cu: the steady-state kernel with the phases ordered by input arrival (one warp per env)
      const int stride = phc::fast::env_stride(amp_dim);
      for (int env = 0; env < a->num_envs; ++env) {
        EmuWarp warp;
        std::vector<std::thread> lanes;
        for (int lane = 0; lane < 32; ++lane)
          lanes.emplace_back([&, lane] {
            emu_warp = &warp;
            emu_lane = lane;
            threadIdx.x = (unsigned)((env % phc::fast::kWarps) * 32 + lane); threadIdx.y = threadIdx.z = 0;
            blockIdx.x = (unsigned)(env / phc::fast::kWarps); blockIdx.y = blockIdx.z = 0;
            phc::fast::env_step_fast_kernel(*a, amp_dim, stride);
          });
        for (auto& t : lanes) t.join();
      }
      return 0;
    }
    case 6:      // env_step_wide.cu: strided bodies, no staging
      for (int env = 0; env < a->num_envs; ++env) {
        EmuWarp warp;
        std::vector<std::thread> lanes;
        for (int lane = 0; lane < 32; ++lane)
          lanes.emplace_back([&, lane] {
            emu_warp = &warp;
            emu_lane = lane;
            threadIdx.x = (unsigned)((env % phc::wide::kWarps) * 32 + lane); threadIdx.y = threadIdx.z = 0;
            blockIdx.x = (unsigned)(env / phc::wide::kWarps); blockIdx.y = blockIdx.z = 0;
            phc::wide::env_step_wide_kernel(*a, obs_dim, self_dim, amp_dim);
          });
        for (auto& t : lanes) t.join();
      }
          return 0;
  }
  return -1;
}
extern "C" uint32_t emu_fast_flags(void) { return phc::kFastFlags; }
'''


def assemble() -> str:
    common = open(os.path.join(CSRC, "phc_common.cuh")).read()
    a = common.index("__device__ __forceinline__ float warp_sum(float v) {")
    b = common.index("}  // namespace phc")
    reductions = common[a:b]
    step = open(os.path.join(CSRC, "env_step.cu")).read()
    k0 = step.index("namespace phc {")
    k1 = step.index("}  // namespace phc") + len("}  // namespace phc")
    kernel = step[k0:k1]
    assert "env_step_kernel(" in kernel and "<<<" not in kernel
    pk = open(os.path.join(CSRC, "env_step_fast.cu")).read()
    p0 = pk.index("namespace phc {")
    p1 = pk.index("}  // namespace phc") + len("}  // namespace phc")
    fastk = pk[p0:p1]
    assert "env_step_fast_kernel(" in fastk and "<<<" not in fastk
    w = open(os.path.join(CSRC, "env_step_wide.cu")).read()
    w0 = w.index("namespace phc {")
    w1 = w.index("}  // namespace phc") + len("}  // namespace phc")
    wide = w[w0:w1]
    assert "env_step_wide_kernel(" in wide and "<<<" not in wide
    return "\n".join([
        '#include "cuda_emu_prelude.h"', '#include "phc_common_emu.cuh"',
        "namespace phc {", reductions, "}",
        f'#include "{os.path.join(ROOT, "include", "phc_b200.h")}"', f'#include "{os.path.join(CSRC, "phc_math.cuh")}"',
        f'#include "{os.path.join(CSRC, "env_step_shared.cuh")}"',
        kernel, fastk, wide, LAUNCHER])


MOTION_LAUNCHER = r'''
template <class F>
static void emu_warps(int64_t n_warps, F&& body) {      // one warp (32 threads) at a time, 4 warps per block like the launches
  for (int64_t w = 0; w < n_warps; ++w) {
    EmuWarp warp;
    std::vector<std::thread> lanes;
    for (int lane = 0; lane < 32; ++lane)
      lanes.emplace_back([&, lane] {
        emu_warp = &warp;
        emu_lane = lane;
        blockDim.x = 128; blockDim.y = blockDim.z = 1;
        threadIdx.x = (unsigned)((w % 4) * 32 + lane); threadIdx.y = threadIdx.z = 0;
        blockIdx.x = (unsigned)(w / 4); blockIdx.y = blockIdx.z = 0;
        body();
      });
    for (auto& t : lanes) t.join();
  }
}

extern "C" int emu_motion_state(const PhcMotionLib* lib, const int64_t* ids, const float* times, const float* offset, int64_t n,
                                const PhcMotionStateOut* out, int wide) {
  if (wide) emu_warps(n, [&] { phc::wide::motion_state_wide_kernel(*lib, ids, times, offset, n, *out); });
  else emu_warps(n, [&] { phc::motion_state_kernel(*lib, ids, times, offset, n, *out); });
  return 0;
}

extern "C" int emu_amp_obs_demo(const PhcMotionLib* lib, const int64_t* ids, const float* times0, int64_t n, int32_t first_step,
                                int32_t num_steps, float dt, uint32_t flags, const int32_t* key_bodies, int32_t nk,
                                const int32_t* amp_joints, int32_t nj, float* out, int64_t out_stride, const int64_t* only_where,
                                int32_t slot_offset, int wide) {
  const int32_t so = ((slot_offset % num_steps) + num_steps) % num_steps;
  if (wide) {
    phc::wide::AmpDemoWideArgs a;
    a.lib = *lib; a.ids = ids; a.times0 = times0; a.n = n; a.first_step = first_step; a.num_steps = num_steps; a.dt = dt;
    a.flags = flags; a.num_key_bodies = nk; a.num_amp_joints = nj; a.out = out; a.out_stride = out_stride; a.only_where = only_where;
    for (int i = 0; i < PHC_MAX_AMP_JOINTS; ++i) a.amp_joints[i] = i < nj ? amp_joints[i] : -1;
    for (int i = 0; i < PHC_MAX_KEY_BODIES; ++i) a.key_bodies[i] = i < nk ? key_bodies[i] : -1;
    a.slot_offset = so; a.slot_offset_dev = nullptr;
    emu_warps(n * num_steps, [&] { phc::wide::amp_demo_wide_kernel(a); });
  } else {
    phc::AmpDemoArgs a;
    a.lib = *lib; a.ids = ids; a.times0 = times0; a.n = n; a.first_step = first_step; a.num_steps = num_steps; a.dt = dt;
    a.flags = flags; a.num_key_bodies = nk; a.num_amp_joints = nj; a.out = out; a.out_stride = out_stride; a.only_where = only_where;
    for (int i = 0; i < PHC_MAX_AMP_JOINTS; ++i) a.amp_joints[i] = i < nj ? amp_joints[i] : -1;
    for (int i = 0; i < PHC_MAX_KEY_BODIES; ++i) a.key_bodies[i] = i < nk ? key_bodies[i] : -1;
    a.slot_offset = so; a.slot_offset_dev = nullptr;
    emu_warps(n * num_steps, [&] { phc::amp_demo_kernel(a); });
  }
  return 0;
}

extern "C" int emu_set_env_state(const PhcMotionLib* lib, const int64_t* ids, const float* times, const float* offset,
                                 const int64_t* only_where, int64_t n, float* body_state, int32_t bpe, float* dof_state, int wide) {
  if (wide) emu_warps(n, [&] { phc::wide::set_env_state_wide_kernel(*lib, ids, times, offset, only_where, n, body_state, bpe, dof_state); });
  else emu_warps(n, [&] { phc::set_env_state_kernel(*lib, ids, times, offset, only_where, n, body_state, bpe, dof_state); });
  return 0;
}
'''


def assemble_motion() -> str:
    """motion.cu (lane-per-body kernels) + motion_wide.cu (strided kernels) + the shared motion_sample.cuh, verbatim."""
    def kernels(fname):
        t = open(os.path.join(CSRC, fname)).read()
        k0 = t.index("namespace phc {")
        k1 = t.index("}  // namespace phc") + len("}  // namespace phc")
        body = t[k0:k1]
        assert "<<<" not in body
        return body
    m = kernels("motion.cu")
    # the pack / gather / bookkeeping / export kernels use plain thread indexing (no warp structure): not emulated here
    return "\n".join([
        '#include "cuda_emu_prelude.h"', '#include "phc_common_emu.cuh"',
        f'#include "{os.path.join(ROOT, "include", "phc_b200.h")}"', f'#include "{os.path.join(CSRC, "phc_math.cuh")}"',
        f'#include "{os.path.join(CSRC, "motion_sample.cuh")}"',
        m, kernels("motion_wide.cu"), MOTION_LAUNCHER])


def build_motion(out_dir: str) -> str:
    gxx = shutil.which("g++")
    if gxx is None:
        raise RuntimeError("g++ not available")
    src = os.path.join(out_dir, "motion_emu.cpp")
    with open(src, "w") as f:
        f.write(assemble_motion())
    so = os.path.join(out_dir, "libmotion_emu.so")
    r = subprocess.run([gxx, "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + HERE, src, "-o", so, "-lm"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("motion emulation build failed:\n" + r.stderr[:6000])
    return so


LOAD_LAUNCHER = r'''
namespace phc { namespace load { alignas(16) unsigned char smem_raw[1 << 17]; } }     // the kernel's dynamic shared memory

extern "C" int emu_motion_load(const double* quat, const double* trans, const double* offsets, const int32_t* parents, const double* heading,
                               const int64_t* starts, const int64_t* nframes, const double* fps, int64_t F, int32_t M, int32_t J, float* gts,
                               float* grs, float* lrs, float* gvs, float* gavs, float* dvs, double* pos64, double* rawang, int32_t* frame_clip) {
  using namespace phc::load;
  FkArgs fa;
  fa.quat = quat; fa.trans = trans; fa.offsets = offsets; fa.parents = parents; fa.heading = heading; fa.starts = starts; fa.nframes = nframes;
  fa.fps = fps; fa.F = F; fa.M = M; fa.J = J; fa.gts = gts; fa.grs = grs; fa.lrs = lrs; fa.dvs = dvs; fa.pos64 = pos64; fa.rawang = rawang;
  fa.frame_clip = frame_clip;
  for (int64_t f = 0; f < F; ++f) {                 // motion_fk_kernel: one warp per frame, kWarps warps per block
    EmuWarp warp;
    std::vector<std::thread> lanes;
    for (int lane = 0; lane < 32; ++lane)
      lanes.emplace_back([&, lane] {
        emu_warp = &warp;
        emu_lane = lane;
        blockDim.x = kWarps * 32;
        threadIdx.x = (unsigned)((f % kWarps) * 32 + lane); blockIdx.x = (unsigned)(f / kWarps);
        motion_fk_kernel(fa);
      });
    for (auto& t : lanes) t.join();
  }
  FilterArgs fl;
  fl.pos64 = pos64; fl.rawang = rawang; fl.frame_clip = frame_clip; fl.starts = starts; fl.nframes = nframes; fl.fps = fps; fl.F = F; fl.J = J;
  fl.gvs = gvs; fl.gavs = gavs;
  {   // the taps exactly as phc_motion_load builds them
    double sum = 0.0;
    for (int k = -kRadius; k <= kRadius; ++k) { fl.taps.w[k + kRadius] = exp(-0.5 / (2.0 * 2.0) * (double)k * (double)k); sum += fl.taps.w[k + kRadius]; }
    for (int k = 0; k <= 2 * kRadius; ++k) fl.taps.w[k] /= sum;
  }
  blockDim.x = 256;                                 // motion_filter_kernel: one thread per (frame, body), no cooperation
  for (int64_t i = 0; i < F * J; ++i) { blockIdx.x = (unsigned)(i / 256); threadIdx.x = (unsigned)(i % 256); motion_filter_kernel(fl); }
  return 0;
}
'''


def build_load(out_dir: str) -> str:
    """motion_load.cu (the loader kernels), verbatim."""
    gxx = shutil.which("g++")
    if gxx is None:
        raise RuntimeError("g++ not available")
    t = open(os.path.join(CSRC, "motion_load.cu")).read()
    k0 = t.index("namespace phc {")
    k1 = t.index("}  // namespace phc") + len("}  // namespace phc")
    body = t[k0:k1]
    assert "<<<" not in body and "motion_fk_kernel" in body
    src = os.path.join(out_dir, "motion_load_emu.cpp")
    with open(src, "w") as f:
        f.write("\n".join(['#include "cuda_emu_prelude.h"', '#include "phc_common_emu.cuh"', "using std::max; using std::min;",
                           f'#include "{os.path.join(ROOT, "include", "phc_b200.h")}"', f'#include "{os.path.join(CSRC, "phc_math.cuh")}"',
                           body, LOAD_LAUNCHER]))
    so = os.path.join(out_dir, "libmotion_load_emu.so")
    r = subprocess.run([gxx, "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + HERE, src, "-o", so, "-lm"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("loader emulation build failed:\n" + r.stderr[:6000])
    return so


SCALARS_LAUNCHER = r'''
template <class F>
static void emu_blocks(int grid, int threads, F&& body) {     // block-level kernels: every thread of a block runs concurrently
  for (int b = 0; b < grid; ++b) {
    std::vector<EmuWarp> warps((threads + 31) / 32);
    std::barrier<> block_bar(threads);
    emu_block_bar = &block_bar;
    std::vector<std::thread> ts;
    for (int t = 0; t < threads; ++t)
      ts.emplace_back([&, t] {
        emu_warp = &warps[t / 32];
        emu_lane = t % 32;
        blockDim.x = (unsigned)threads; gridDim.x = (unsigned)grid;
        threadIdx.x = (unsigned)t; blockIdx.x = (unsigned)b;
        body();
      });
    for (auto& t : ts) t.join();
  }
  emu_block_bar = nullptr;
}

extern "C" int emu_gae(const float* fdones, const float* values, const float* rewards, const float* next_values, int32_t T, int64_t N,
                       float gamma, float tau, float* advs, float* returns) {
  emu_blocks((int)((N + 31) / 32), 1024, [&] { phc::gae_kernel(fdones, values, rewards, next_values, T, N, gamma, tau, advs, returns); });
  return 0;
}

extern "C" int emu_adv_norm(const float* returns, const float* values, int64_t n, int32_t normalize, float* advs, double* workspace) {
  const int g = phc::adv_grid(n);
  emu_blocks(g, phc::kAdvBlock, [&] { phc::adv_partial_kernel(returns, values, n, advs, workspace); });
  if (normalize) emu_blocks(g, phc::kAdvBlock, [&] { phc::adv_apply_kernel(advs, n, workspace, g); });
  return g;
}
'''


def build_scalars(out_dir: str) -> str:
    """ppo_scalars.cu (GAE scan, advantage normalisation), verbatim; `__shared__` variables become function-local statics."""
    gxx = shutil.which("g++")
    if gxx is None:
        raise RuntimeError("g++ not available")
    t = open(os.path.join(CSRC, "ppo_scalars.cu")).read()
    k0 = t.index("namespace phc {")
    k1 = t.index("}  // namespace phc") + len("}  // namespace phc")
    body = t[k0:k1]
    assert "<<<" not in body and "gae_kernel" in body
    src = os.path.join(out_dir, "ppo_scalars_emu.cpp")
    with open(src, "w") as f:
        f.write("\n".join(['#include "cuda_emu_prelude.h"', "#undef __shared__", "#define __shared__ static",
                           f'#include "{os.path.join(ROOT, "include", "phc_b200.h")}"', body, SCALARS_LAUNCHER]))
    so = os.path.join(out_dir, "libppo_scalars_emu.so")
    r = subprocess.run([gxx, "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + HERE, src, "-o", so, "-lm"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("ppo_scalars emulation build failed:\n" + r.stderr[:6000])
    return so


UPDATE_LAUNCHER = r'''
template <class F>
static void emu_grid(int gx, int gy, int bx, int by, F&& body) {     // 2-D grids / blocks, every thread of a block concurrent
  const int threads = bx * by;
  for (int b = 0; b < gx * gy; ++b) {
    std::vector<EmuWarp> warps((threads + 31) / 32);
    std::barrier<> block_bar(threads);
    emu_block_bar = &block_bar;
    std::vector<std::thread> ts;
    for (int t = 0; t < threads; ++t)
      ts.emplace_back([&, t] {
        emu_warp = &warps[t / 32];
        emu_lane = t % 32;
        blockDim.x = (unsigned)bx; blockDim.y = (unsigned)by; gridDim.x = (unsigned)gx; gridDim.y = (unsigned)gy;
        threadIdx.x = (unsigned)(t % bx); threadIdx.y = (unsigned)(t / bx); blockIdx.x = (unsigned)(b % gx); blockIdx.y = (unsigned)(b / gx);
        body();
      });
    for (auto& t : ts) t.join();
  }
  emu_block_bar = nullptr;
}

extern "C" int emu_rms_apply(const float* x, int64_t ldx, int64_t n, int32_t d, const double* mean, const double* var, float eps, int32_t unnorm,
                             float* y, int64_t ldy, const int64_t* row_idx) {
  emu_grid(2, 1, 256, 1, [&] { phc::rms_apply_kernel(x, ldx, n, d, mean, var, eps, unnorm, y, ldy, row_idx); });      // grid-stride: any grid
  return 0;
}
extern "C" int emu_rms_update(const float* x, int64_t ldx, int64_t n, int32_t d, double* mean, double* var, double* count, double* acc,
                              const int64_t* row_idx) {
  int gy = (int)((n + 1023) / 1024); if (gy > 32) gy = 32; if (gy < 1) gy = 1;
  emu_grid((d + 31) / 32, gy, 32, 32, [&] { phc::rms_moments_kernel(x, ldx, n, d, acc, row_idx); });
  emu_grid(1, 1, 1024, 1, [&] { phc::rms_merge_kernel(acc, gy, n, d, mean, var, count); });
  return 0;
}
extern "C" int emu_rms_apply_update_vec(const float* x, int64_t ldx, int64_t n, int32_t d, const double* mean_a, const double* var_a, float eps,
                                       float* y, int64_t ldy, const int64_t* row_idx, double* mean, double* var, double* count, double* acc,
                                       int32_t V, int32_t rows_per_block, int32_t moments) {
  const int cb = (d + 32 * V - 1) / (32 * V), gy = (int)((n + rows_per_block - 1) / rows_per_block);
  emu_grid(cb, gy, 256, 1, [&] {
    if (V == 4 && moments) phc::rms_apply_vec_kernel<4, true>(x, ldx, n, d, mean_a, var_a, eps, y, ldy, row_idx, acc, rows_per_block);
    else if (V == 4) phc::rms_apply_vec_kernel<4, false>(x, ldx, n, d, mean_a, var_a, eps, y, ldy, row_idx, nullptr, rows_per_block);
    else if (moments) phc::rms_apply_vec_kernel<2, true>(x, ldx, n, d, mean_a, var_a, eps, y, ldy, row_idx, acc, rows_per_block);
    else phc::rms_apply_vec_kernel<2, false>(x, ldx, n, d, mean_a, var_a, eps, y, ldy, row_idx, nullptr, rows_per_block);
  });
  if (moments) emu_grid(1, 1, 1024, 1, [&] { phc::rms_merge_kernel(acc, gy, n, d, mean, var, count); });
  return 0;
}
extern "C" int emu_disc_reward(const float* logit, int64_t ld, const float* task, int64_t n, float scale, float w_task, float w_disc,
                               float* disc_r, float* combined) {
  emu_grid(2, 1, 256, 1, [&] { phc::disc_reward_kernel(logit, ld, task, n, scale, w_task, w_disc, disc_r, combined); });
  return 0;
}
extern "C" int emu_ppo_actor_grad(const float* mu, int64_t ldmu, const float* logstd, const float* actions, const float* old_neglogp, const float* adv,
                                  const float* old_mu, const float* old_sigma, int64_t n, int32_t A, float e_clip, float bound_coef, float inv_batch,
                                  float* dmu, int64_t lddmu, float* stats) {
  emu_grid(3, 1, 256, 1, [&] { phc::ppo_actor_grad_kernel(mu, ldmu, logstd, actions, old_neglogp, adv, old_mu, old_sigma, n, A, e_clip, bound_coef,
                                                          inv_batch, dmu, lddmu, stats); });
  return 0;
}
extern "C" int emu_ppo_critic_grad(const float* v, int64_t ldv, const float* ret, int64_t n, float coef, float inv_batch, float* dv, int64_t lddv, float* stats) {
  emu_grid(2, 1, 256, 1, [&] { phc::ppo_critic_grad_kernel(v, ldv, ret, n, coef, inv_batch, dv, lddv, stats); });
  return 0;
}
extern "C" int emu_disc_logit_grad(const float* logit, int64_t ld, int64_t n_agent, int64_t n_demo, float coef, float* dlogit, int64_t ldd, float* stats) {
  emu_grid(2, 1, 256, 1, [&] { phc::disc_logit_grad_kernel(logit, ld, n_agent, n_demo, coef, dlogit, ldd, stats); });
  return 0;
}
extern "C" int emu_clip_adam(float* p, const float* g, float* m, float* v, int64_t n, double* sumsq, float grad_scale, float max_norm, float lr,
                             float beta1, float beta2, float eps, int64_t step) {
  double part[2];
  emu_grid(2, 1, 256, 1, [&] { phc::sumsq_kernel(g, n, part); });
  phc::sum_parts_kernel(part, 2, sumsq);
  const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);      // as phc_adam_step
  emu_grid(2, 1, 256, 1, [&] { phc::adam_clip_kernel(p, g, m, v, n, sumsq, grad_scale, max_norm, lr, beta1, beta2, eps, (float)bc1, (float)sqrt(bc2)); });
  return 0;
}
extern "C" int emu_mcp_combine(const float* w, int64_t ldw, const float* prim, int64_t ldp, int64_t prim_stride, int64_t n, int32_t K, int32_t A,
                               int32_t discrete, float* out, int64_t ldo) {
  emu_grid(2, 1, 256, 1, [&] { phc::mcp_combine_kernel(w, ldw, prim, ldp, prim_stride, n, K, A, discrete, out, ldo); });
  return 0;
}
extern "C" int emu_gaussian_sample(const float* mu, int64_t ldmu, const float* logstd, const float* noise, int64_t n, int32_t A, float* actions,
                                   float* neglogp, float* mus, float* sigmas) {
  emu_grid((int)((n + 3) / 4), 1, 128, 1, [&] { phc::gaussian_sample_kernel(mu, ldmu, logstd, noise, n, A, actions, neglogp, mus, sigmas); });
  return 0;
}
'''


def build_update(out_dir: str) -> str:
    """ppo_update.cu (RunningMeanStd, Gaussian head, losses, optimiser kernels), verbatim; a few of them get launchers here."""
    gxx = shutil.which("g++")
    if gxx is None:
        raise RuntimeError("g++ not available")
    t = open(os.path.join(CSRC, "ppo_update.cu")).read()
    k0 = t.index("namespace phc {")
    k1 = t.index("}  // namespace phc") + len("}  // namespace phc")
    body = t[k0:k1]
    assert "<<<" not in body and "rms_apply_kernel" in body
    src = os.path.join(out_dir, "ppo_update_emu.cpp")
    with open(src, "w") as f:
        f.write("\n".join(['#include "cuda_emu_prelude.h"', "#undef __shared__", "#define __shared__ static",
                           f'#include "{os.path.join(ROOT, "include", "phc_b200.h")}"',
                           "namespace phc { static inline float silu_f(float x) { return x / (1.0f + expf(-x)); }",
                           "static inline float silu_grad_f(float z) { const float sg = 1.0f / (1.0f + expf(-z)); return sg * (1.0f + z * (1.0f - sg)); } }",
                           body, UPDATE_LAUNCHER]))
    so = os.path.join(out_dir, "libppo_update_emu.so")
    r = subprocess.run([gxx, "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + HERE, src, "-o", so, "-lm"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("ppo_update emulation build failed:\n" + r.stderr[:8000])
    return so


def build(out_dir: str) -> str:
    gxx = shutil.which("g++")
    if gxx is None:
        raise RuntimeError("g++ not available")
    src = os.path.join(out_dir, "env_step_emu.cpp")
    with open(src, "w") as f:
        f.write(assemble())
    so = os.path.join(out_dir, "libenv_step_emu.so")
    r = subprocess.run([gxx, "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + HERE, src, "-o", so, "-lm"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("emulation build failed:\n" + r.stderr[:6000])
    return so


if __name__ == "__main__":
    import tempfile
    d = tempfile.mkdtemp()
    print(build(d))
    print(build_motion(d))
    print(build_load(d))
    print(build_scalars(d))
    print(build_update(d))
