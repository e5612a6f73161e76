"""TEST INFRASTRUCTURE: the CPU emulation of build_emu.py for the get-up schedule: the recovery instantiations of env_step_kernel
(REC = true: SMPL, generic run-time J, keypoint) and of the strided kernel, plus the two kernels of getup.cu (phc_getup_reset's
single-CTA selection and its state copy, phc_amp_ring_fill), all verbatim product source.  The selection kernel runs as one block of
1024 concurrent threads (`__syncthreads` = a block barrier, `__shared__` = one copy per block)."""
import ctypes as C
import os
import shutil
import subprocess

import build_emu
from host_plan import round4

from phc_b200 import _lib

EXTRA_PRELUDE = r'''
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __shfl_up_sync(unsigned, int v, int o) { return emu_exchange(v, emu_lane - o); }
'''

LAUNCHER = r'''
template <int JT, bool KP>
static void emu_launch_rec(const PhcStepArgs& a, int obs_dim, int self_dim, int amp_dim, bool alias_obs, bool state_bulk_ok) {
  for (int env = 0; env < a.num_envs; ++env) {
    EmuWarp warp;
    std::vector<std::thread> lanes;
    for (int lane = 0; lane < 32; ++lane)
      lanes.emplace_back([&, lane] {
        emu_warp = &warp;
        emu_lane = lane;
        threadIdx.x = (unsigned)((env % phc::kWarpsPerCta) * 32 + lane); threadIdx.y = threadIdx.z = 0;
        blockIdx.x = (unsigned)(env / phc::kWarpsPerCta); blockIdx.y = blockIdx.z = 0;
        phc::env_step_kernel<1, JT, true, false, KP, true>(a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok);
      });
    for (auto& t : lanes) t.join();
  }
}

extern "C" int emu_env_step_rec(const PhcStepArgs* a, int obs_dim, int self_dim, int amp_dim, int alias_obs, int state_bulk_ok, int variant) {
  switch (variant) {
    case 0: emu_launch_rec<24, false>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 1: emu_launch_rec<0, false>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 2: emu_launch_rec<24, true>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 3:      // the strided kernel's recovery instantiation
      for (int env = 0; env < a->num_envs; ++env) {
        EmuWarp warp;
        std::vector<std::thread> lanes;
        for (int lane = 0; lane < 32; ++lane)
          lanes.emplace_back([&, lane] {
            emu_warp = &warp;
            emu_lane = lane;
            threadIdx.x = (unsigned)((env % phc::wide::kWarps) * 32 + lane); threadIdx.y = threadIdx.z = 0;
            blockIdx.x = (unsigned)(env / phc::wide::kWarps); blockIdx.y = blockIdx.z = 0;
            phc::wide::env_step_wide_kernel<true>(*a, obs_dim, self_dim, amp_dim);
          });
        for (auto& t : lanes) t.join();
      }
      return 0;
  }
  return -1;
}

template <class F>
static void emu_blocks(int grid, int threads, F&& body) {          // 1-D grid, every thread of a block concurrent
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
        threadIdx.x = (unsigned)t; threadIdx.y = threadIdx.z = 0; blockIdx.x = (unsigned)b; blockIdx.y = blockIdx.z = 0;
        body();
      });
    for (auto& t : ts) t.join();
  }
  emu_block_bar = nullptr;
}

// phc_getup_reset's two launches (getup.cu), argument for argument
extern "C" void emu_getup_reset(const int64_t* mask, const int64_t* terminate_in, const float* u_rec, const float* u_fall, const int64_t* perm,
                                const float* p_rec, const float* p_fall, int32_t recovery_steps, const float* fall_root, const float* fall_dof_pos,
                                int64_t P, int64_t* available, int64_t* assignment, int32_t* counter, int64_t n, float* body_state,
                                int32_t bodies_per_env, float* dof_state, int32_t D, int64_t* progress, int64_t* reset, int64_t* terminate,
                                int64_t* ref_init, int64_t* fall) {
  using namespace phc::getup;
  emu_blocks(1, kThreads, [&] {
    select_kernel(mask, terminate_in, u_rec, u_fall, perm, p_rec, p_fall, recovery_steps, P, available, assignment, counter, n, progress, reset,
                  terminate, ref_init, fall);
  });
  emu_blocks((int)((n + kCopyWarps - 1) / kCopyWarps), kCopyWarps * 32, [&] {
    copy_kernel(fall, assignment, fall_root, fall_dof_pos, n, body_state, bodies_per_env, dof_state, D);
  });
}

extern "C" void emu_amp_ring_fill(float* ring, int64_t stride, int64_t n, int32_t S, int32_t A, const int32_t* head, const int64_t* mask) {
  using namespace phc::getup;
  emu_blocks((int)((n + kCopyWarps - 1) / kCopyWarps), kCopyWarps * 32, [&] { ring_fill_kernel(ring, stride, n, S, A, head, mask); });
}
'''


def assemble() -> str:
    t = open(os.path.join(build_emu.CSRC, "getup.cu")).read()
    k0 = t.index("namespace phc {")
    k1 = t.index("}  // namespace phc") + len("}  // namespace phc")
    getup = t[k0:k1]
    assert "select_kernel(" in getup and "<<<" not in getup
    return "\n".join([build_emu.assemble(), EXTRA_PRELUDE, "#undef __shared__", "#define __shared__ static", getup, LAUNCHER])


def build(out_dir: str) -> str:
    gxx = shutil.which("g++")
    if gxx is None:
        raise RuntimeError("g++ not available")
    src = os.path.join(out_dir, "getup_emu.cpp")
    with open(src, "w") as f:
        f.write(assemble())
    so = os.path.join(out_dir, "libgetup_emu.so")
    r = subprocess.run([gxx, "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + build_emu.HERE, src, "-o", so,
                        "-lm"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("emulation build failed:\n" + r.stderr[:6000])
    return so


class EmuGetup:
    # the instantiations phc_env_step launches for PHC_FLAG_RECOVERY / PHC_FLAG_AMP_CURRENT
    VARIANTS = {"smpl": 0, "generic": 1, "kp": 2, "wide": 3}

    def __init__(self, so_path):
        self.lib = C.CDLL(so_path)
        self.lib.emu_env_step_rec.restype = C.c_int
        self.lib.emu_env_step_rec.argtypes = [C.POINTER(_lib.PhcStepArgs)] + [C.c_int] * 6
        p = C.c_void_p
        self.lib.emu_getup_reset.restype = None
        self.lib.emu_getup_reset.argtypes = [p, p, p, p, p, p, p, C.c_int32, p, p, C.c_int64, p, p, p, C.c_int64, p, C.c_int32, p, C.c_int32,
                                             p, p, p, p, p]
        self.lib.emu_amp_ring_fill.restype = None
        self.lib.emu_amp_ring_fill.argtypes = [p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, p, p]

    def run(self, plan, variant):
        a = plan.args
        assert a.flags & (_lib.PHC_FLAG_RECOVERY | _lib.PHC_FLAG_AMP_CURRENT)
        J = a.lib.num_bodies
        obs_dim, self_dim = plan.obs_dim, plan.self_dim
        alias_obs = 2 * a.lib.body_stride + round4(J * 13) >= round4(obs_dim)
        state_bulk_ok = (a.body_state % 16 == 0) and ((a.bodies_per_env * 13) % 4 == 0) and ((J * 13) % 4 == 0)
        rc = self.lib.emu_env_step_rec(C.byref(a), obs_dim, self_dim, plan.amp_dim if a.amp_out else 0, int(alias_obs), int(state_bulk_ok),
                                       self.VARIANTS[variant])
        assert rc == 0

    def getup_reset(self, mask, term_in, u_rec, u_fall, perm, probs, steps, fall_root, fall_dof, available, assignment, counter, body_state,
                    dof_state, progress, reset, term, ref_init, fall):
        """ops.getup_reset's arguments as host tensors (contiguous, the dtypes of the C ABI)."""
        ptr = lambda t: t.data_ptr()
        n, P = mask.shape[0], fall_root.shape[0]
        self.lib.emu_getup_reset(ptr(mask), ptr(term_in), ptr(u_rec), ptr(u_fall), ptr(perm), ptr(probs), probs.data_ptr() + 4, int(steps),
                                 ptr(fall_root), ptr(fall_dof), P, ptr(available), ptr(assignment), ptr(counter), n, ptr(body_state),
                                 body_state.shape[1], ptr(dof_state), dof_state.shape[1], ptr(progress), ptr(reset), ptr(term),
                                 ptr(ref_init), ptr(fall))

    def amp_ring_fill(self, ring, mask):
        n, S, A = ring.shape
        self.lib.emu_amp_ring_fill(ring.data_ptr(), ring.stride(0), n, S, A, None, mask.data_ptr())
