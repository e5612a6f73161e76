"""TEST INFRASTRUCTURE: the CPU emulation of build_emu.py (the env-step kernel source, verbatim) with launchers for the keypoint
instantiations of env_step_kernel (KP = true, PHC_FLAG_TASK_OBS_KP), driven like host_plan.Emu."""
import ctypes as C
import os
import shutil
import subprocess

import build_emu
from host_plan import round4

from phc_b200 import _lib

KP_LAUNCHER = r'''
template <int T_MAX, int JT, bool GETUP>
static void emu_launch_kp(const PhcStepArgs& a, int obs_dim, int self_dim, int amp_dim, bool alias_obs, bool state_bulk_ok) {
  for (int env = 0; env < a.num_envs; ++env) {
    EmuWarp warp;
    std::vector<std::thread> lanes;
    for (int lane = 0; lane < 32; ++lane)
      lanes.emplace_back([&, lane] {
        emu_warp = &warp;
        emu_lane = lane;
        threadIdx.x = (unsigned)((env % phc::kWarpsPerCta) * 32 + lane); threadIdx.y = threadIdx.z = 0;
        blockIdx.x = (unsigned)(env / phc::kWarpsPerCta); blockIdx.y = blockIdx.z = 0;
        phc::env_step_kernel<T_MAX, JT, GETUP, false, true>(a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok);
      });
    for (auto& t : lanes) t.join();
  }
}

extern "C" int emu_env_step_kp(const PhcStepArgs* a, int obs_dim, int self_dim, int amp_dim, int alias_obs, int state_bulk_ok, int variant) {
  switch (variant) {
    case 0: emu_launch_kp<1, 24, false>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 1: emu_launch_kp<1, 24, true>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 2: emu_launch_kp<1, 0, false>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
    case 3: emu_launch_kp<4, 0, false>(*a, obs_dim, self_dim, amp_dim, alias_obs, state_bulk_ok); return 0;
  }
  return -1;
}
'''


def build(out_dir: str) -> str:
    gxx = shutil.which("g++")
    if gxx is None:
        raise RuntimeError("g++ not available")
    src = os.path.join(out_dir, "env_step_kp_emu.cpp")
    with open(src, "w") as f:
        f.write(build_emu.assemble() + KP_LAUNCHER)
    so = os.path.join(out_dir, "libenv_step_kp_emu.so")
    r = subprocess.run([gxx, "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + build_emu.HERE, src, "-o", so,
                        "-lm"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("emulation build failed:\n" + r.stderr[:6000])
    return so


class EmuKp:
    # the instantiations phc_env_step launches for PHC_FLAG_TASK_OBS_KP
    VARIANTS = {"smpl": 0, "getup": 1, "generic": 2, "fut": 3}

    def __init__(self, so_path):
        self.lib = C.CDLL(so_path)
        self.lib.emu_env_step_kp.restype = C.c_int
        self.lib.emu_env_step_kp.argtypes = [C.POINTER(_lib.PhcStepArgs)] + [C.c_int] * 6

    def run(self, plan, variant):
        a = plan.args
        assert a.flags & _lib.PHC_FLAG_TASK_OBS_KP
        J = a.lib.num_bodies
        # the launcher's derived arguments (phc_env_step in env_step.cu), from the plan's sizes (EnvStepPlan asks the library)
        obs_dim, self_dim = plan.obs_dim, plan.self_dim
        alias_obs = 2 * a.lib.body_stride + round4(J * 13) >= round4(obs_dim)
        state_bulk_ok = (a.body_state % 16 == 0) and ((a.bodies_per_env * 13) % 4 == 0) and ((J * 13) % 4 == 0)
        rc = self.lib.emu_env_step_kp(C.byref(a), obs_dim, self_dim, plan.amp_dim if a.amp_out else 0, int(alias_obs), int(state_bulk_ok),
                                      self.VARIANTS[variant])
        assert rc == 0
