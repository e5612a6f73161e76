"""Timing of the evaluation metrics on the GPU, in one process:
  * phc_eval_metrics_step alone: CUDA events around `iters` back-to-back launches (every frame counted, so the Procrustes solve runs
    for every env), at 4096 and 16384 envs, J = 24 and 52, body positions read as the [..., :J, 0:3] view of a [N, J, 13] state;
    the bytes it has to move (positions, reference positions, two ring slots read and one written, the fp64 accumulator row read and
    written) over that time;
  * one whole IMAmpAgent.eval() sweep at 4096 envs (4096 clips, one batch) on a SyntheticSim-based owner that tracks the reference
    pose, with `full_eval_metrics` on and off, alternated, host wall time around the call (ends in a device synchronise).
Prints the card name and power limit with the numbers.
    python tools/time_eval_metrics.py [iters]"""
import json
import os
import statistics
import subprocess
import sys
import time
from types import SimpleNamespace

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from phc_b200 import ops, synthetic as syn  # noqa: E402
from phc_b200.env.humanoid_im import HumanoidIm, RLGPUEnv, SyntheticSim  # noqa: E402
from phc_b200.learning.im_amp import IMAmpAgent  # noqa: E402

DEV = "cuda:0"


def time_kernel(n, J, iters):
    g = torch.Generator(device=DEV).manual_seed(n + J)
    state = torch.randn(n, J, 13, device=DEV, generator=g)
    gt = (state[..., 0:3] + 0.05 * torch.randn(n, J, 3, device=DEV, generator=g)).contiguous()
    steps = torch.full((n,), 1 << 30, dtype=torch.int32, device=DEV)
    ring = torch.zeros(2, n, J, 3, device=DEV)
    acc = torch.zeros(n, 8, dtype=torch.float64, device=DEV)
    pos = state[..., 0:3]
    for t in range(10):
        ops.eval_metrics_step(pos, gt, steps, t, ring, acc)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(iters):
        ops.eval_metrics_step(pos, gt, steps, 10 + t, ring, acc)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    nbytes = n * J * 12 * 5 + n * 64 * 2
    return {"num_envs": n, "J": J, "kernel_us": round(us, 2), "bytes": nbytes, "GB_per_s": round(nbytes / us / 1e3, 1)}


class TrackingSim(SyntheticSim):
    """SyntheticSim with the per-env asset data the motion loader needs; in eval mode simulate() puts the bodies at the reference
    pose plus 2 cm of noise, so no clip terminates and the sweep runs every clip to its end."""

    def __init__(self, num_envs, J=24):
        super().__init__(syn.make_motions(8, seed=1, min_frames=20, max_frames=30), num_envs, DEV, seed=3)
        rng = np.random.default_rng(0)
        off = rng.standard_normal((J, 3)) * 0.15
        off[0] = 0
        self.J = J
        self.skeleton_trees = [SimpleNamespace(local_translation=off, parent_indices=np.array(syn.SMPL_PARENTS, dtype=np.int32),
                                               node_names=[f"b{j}" for j in range(J)]) for _ in range(num_envs)]
        self.humanoid_shapes = torch.zeros(num_envs, 17)
        self.humanoid_limb_and_weights = torch.zeros(num_envs, 10)
        self.pd_action_offset = torch.zeros(3 * (J - 1))
        self.pd_action_scale = torch.full((3 * (J - 1),), 1.5)
        self.task = None

    def simulate(self, actions):
        super().simulate(actions)
        task = self.task
        if task is None or not getattr(task, "_eval_mode", False):
            return
        t = (task.progress_buf + 1).float() * task.dt + task._motion_start_times + task._motion_start_times_offset
        pos = ops.motion_state(task._motion_lib, task._sampled_motion_ids, t.contiguous(), task._global_offset.contiguous(), want_dof=False)["rg_pos"]
        self.rigid_body_state[:, :self.J, 0:3] = pos + 0.02 * torch.randn_like(pos)


def make_clips(M, J, seed):
    rng = np.random.default_rng(seed)
    clips = {}
    for i in range(M):
        n = int(rng.integers(30, 61))
        w = np.cumsum(rng.standard_normal((n, J, 4)) * 0.05, 0) + rng.standard_normal((1, J, 4))
        clips[f"clip{i}"] = {"pose_quat_global": w / np.linalg.norm(w, axis=-1, keepdims=True),
                             "root_trans_offset": torch.from_numpy(np.cumsum(rng.standard_normal((n, 3)) * 0.02, 0)),
                             "pose_aa": np.zeros((n, 72)), "fps": 30.0}
    return clips


def time_sweeps(n, reps):
    sim = TrackingSim(n)
    cfg = {"env": {"num_envs": n, "motion_file": make_clips(n, 24, seed=7), "episode_length": 300, "controlFrequencyInv": 2,
                   "numAMPObsSteps": 10, "local_root_obs": True, "root_height_obs": True, "enableEarlyTermination": True,
                   "terminationDistance": 0.25, "power_reward": True},
           "robot": {"humanoid_type": "smpl", "has_upright_start": True, "has_dof_subset": True}, "sim": {"dt": 1.0 / 60.0},
           "seed": 0, "headless": True, "sim_backend": sim}
    task = HumanoidIm(cfg=cfg, sim_params=SimpleNamespace(dt=1.0 / 60.0), physics_engine="physx", device_type="cuda", device_id=0, headless=True)
    sim.task = task
    agent = IMAmpAgent("run", {"vec_env": RLGPUEnv(task), "horizon_length": 8, "minibatch_size": 1024, "amp_minibatch_size": 256,
                               "mini_epochs": 1, "amp_obs_demo_buffer_size": 4096, "amp_replay_buffer_size": 4096, "amp_batch_size": 512})
    agent.obs = agent.env_reset()
    steps = []
    real_step = agent.env_eval_step

    def counting_step(env, actions):
        steps[-1] += 1
        return real_step(env, actions)
    agent.env_eval_step = counting_step
    rows = {True: [], False: []}
    for rep in range(reps + 1):
        for full in (False, True):
            agent.full_eval_metrics = full
            steps.append(0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            info = agent.eval()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if rep > 0:                                      # the first pair warms up
                rows[full].append({"sweep_s": dt, "steps": steps[-1], "info": info})
    return [{"num_envs": n, "full_eval_metrics": full, "sweeps": len(r), "steps_per_sweep": r[0]["steps"],
             "median_sweep_ms": round(statistics.median(x["sweep_s"] for x in r) * 1e3, 1),
             "median_ms_per_step": round(statistics.median(x["sweep_s"] / x["steps"] for x in r) * 1e3, 3),
             "eval_info": r[0]["info"]} for full, r in rows.items()]


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1], "iters": iters, "kernel": [], "sweep": []}
    for n in (4096, 16384):
        for J in (24, 52):
            out["kernel"].append(time_kernel(n, J, iters))
    out["sweep"] = time_sweeps(4096, reps=3)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
