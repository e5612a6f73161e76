"""TEST INFRASTRUCTURE: the CPU emulation of tests/emu (cuda_emu_prelude.h) for the episode-statistics kernel: the `namespace phc`
part of phc_b200/csrc/episode_stats.cu, verbatim, with a launcher that runs its single block as kThreads concurrent threads (warps of
32 lanes, a block barrier for __syncthreads)."""
import ctypes as C
import os
import shutil
import subprocess

import build_emu

LAUNCHER = r'''
extern "C" void emu_episode_stats(const float* rewards, const int64_t* dones, int64_t n, float* cur_r, float* cur_l, float* mean, int32_t* size,
                                  int32_t max_size) {
  using namespace phc::epstats;
  std::vector<EmuWarp> warps(kThreads / 32);
  std::barrier<> block_bar(kThreads);
  emu_block_bar = &block_bar;
  std::vector<std::thread> ts;
  for (int t = 0; t < kThreads; ++t)
    ts.emplace_back([&, t] {
      emu_warp = &warps[t / 32];
      emu_lane = t % 32;
      blockDim.x = kThreads; blockDim.y = blockDim.z = 1; gridDim.x = gridDim.y = gridDim.z = 1;
      threadIdx.x = (unsigned)t; threadIdx.y = threadIdx.z = 0; blockIdx.x = blockIdx.y = blockIdx.z = 0;
      episode_stats_kernel(rewards, dones, n, cur_r, cur_l, mean, size, max_size);
    });
  for (auto& th : ts) th.join();
  emu_block_bar = nullptr;
}
'''


def assemble() -> str:
    t = open(os.path.join(build_emu.CSRC, "episode_stats.cu")).read()
    k0 = t.index("namespace phc {")
    k1 = t.index("}  // namespace phc") + len("}  // namespace phc")
    kernel = t[k0:k1]
    assert "episode_stats_kernel(" in kernel and "<<<" not in kernel
    return "\n".join(['#include "cuda_emu_prelude.h"', "#undef __shared__", "#define __shared__ static",
                      f'#include "{os.path.join(build_emu.ROOT, "include", "phc_b200.h")}"', kernel, LAUNCHER])


def build(out_dir: str) -> str:
    gxx = shutil.which("g++")
    if gxx is None:
        raise RuntimeError("g++ not available")
    src = os.path.join(out_dir, "episode_stats_emu.cpp")
    with open(src, "w") as f:
        f.write(assemble())
    so = os.path.join(out_dir, "libepisode_stats_emu.so")
    r = subprocess.run([gxx, "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + build_emu.HERE, src, "-o", so,
                        "-lm"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("emulation build failed:\n" + r.stderr[:6000])
    return so


class EmuEpisodeStats:
    def __init__(self, so_path):
        self.lib = C.CDLL(so_path)
        p = C.c_void_p
        self.lib.emu_episode_stats.restype = None
        self.lib.emu_episode_stats.argtypes = [p, p, C.c_int64, p, p, p, p, C.c_int32]

    def step(self, rewards, dones, cur_r, cur_l, mean, size, games_to_track):
        """ops.episode_stats's arguments as contiguous host tensors."""
        for t in (rewards, dones, cur_r, cur_l, mean, size):
            assert t.is_contiguous()
        self.lib.emu_episode_stats(rewards.data_ptr(), dones.data_ptr(), cur_r.numel(), cur_r.data_ptr(), cur_l.data_ptr(), mean.data_ptr(),
                                   size.data_ptr(), int(games_to_track))
