"""TEST INFRASTRUCTURE: the CPU emulation of tests/emu (cuda_emu_prelude.h) for the evaluation-metrics kernel: the `namespace phc`
part of phc_b200/csrc/eval_metrics.cu, verbatim, with a launcher that runs the whole grid of phc_eval_metrics_step (kWarps envs per
block, the idle warps of the last block included) one warp of 32 concurrent lane threads at a time."""
import ctypes as C
import os
import shutil
import subprocess

import build_emu

LAUNCHER = r'''
extern "C" void emu_eval_metrics_step(const float* pos, int64_t env_stride, int64_t body_stride, const float* gt, const int32_t* num_steps,
                                      int32_t t, int64_t n, int32_t J, float* ring, double* acc) {
  using namespace phc::evalm;
  const int64_t grid = (n + kWarps - 1) / kWarps;
  for (int64_t w = 0; w < grid * kWarps; ++w) {
    EmuWarp warp;
    std::vector<std::thread> lanes;
    for (int lane = 0; lane < 32; ++lane)
      lanes.emplace_back([&, lane] {
        emu_warp = &warp;
        emu_lane = lane;
        threadIdx.x = (unsigned)((w % kWarps) * 32 + lane); threadIdx.y = threadIdx.z = 0;
        blockIdx.x = (unsigned)(w / kWarps); blockIdx.y = blockIdx.z = 0;
        eval_metrics_kernel(pos, env_stride, body_stride, gt, num_steps, t, n, J, ring, acc);
      });
    for (auto& th : lanes) th.join();
  }
}
'''


def assemble() -> str:
    t = open(os.path.join(build_emu.CSRC, "eval_metrics.cu")).read()
    k0 = t.index("namespace phc {")
    k1 = t.index("}  // namespace phc") + len("}  // namespace phc")
    kernel = t[k0:k1]
    assert "eval_metrics_kernel(" in kernel and "<<<" not in kernel
    return "\n".join(['#include "cuda_emu_prelude.h"', f'#include "{os.path.join(build_emu.ROOT, "include", "phc_b200.h")}"', kernel, LAUNCHER])


def build(out_dir: str) -> str:
    gxx = shutil.which("g++")
    if gxx is None:
        raise RuntimeError("g++ not available")
    src = os.path.join(out_dir, "eval_metrics_emu.cpp")
    with open(src, "w") as f:
        f.write(assemble())
    so = os.path.join(out_dir, "libeval_metrics_emu.so")
    r = subprocess.run([gxx, "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + build_emu.HERE, src, "-o", so,
                        "-lm"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("emulation build failed:\n" + r.stderr[:6000])
    return so


class EmuEvalMetrics:
    def __init__(self, so_path):
        self.lib = C.CDLL(so_path)
        p = C.c_void_p
        self.lib.emu_eval_metrics_step.restype = None
        self.lib.emu_eval_metrics_step.argtypes = [p, C.c_int64, C.c_int64, p, p, C.c_int32, C.c_int64, C.c_int32, p, p]

    def step(self, body_pos, body_pos_gt, num_steps, t, ring, acc):
        """ops.eval_metrics_step's arguments as host tensors (body_pos may be a strided view with x, y, z contiguous)."""
        n, J, _ = body_pos.shape
        assert body_pos.stride(2) == 1 and body_pos_gt.is_contiguous() and ring.is_contiguous() and acc.is_contiguous()
        self.lib.emu_eval_metrics_step(body_pos.data_ptr(), body_pos.stride(0), body_pos.stride(1), body_pos_gt.data_ptr(),
                                       num_steps.data_ptr(), int(t), n, J, ring.data_ptr(), acc.data_ptr())
