"""Generate tests/golden/kp.npz: the keypoint-only task observation (env.obs_v: 7) of the UNMODIFIED reference.

Like make_golden.py (whose environment builder, step and writer it uses) it needs the reference checkout and runs the real
HumanoidIm._compute_reward / _compute_reset / _compute_observations with obs_v = 7, i.e. compute_imitation_observations_v7
(phc/env/tasks/humanoid_im.py:1362-1393) reached through _compute_task_obs (:832-853).  The inputs are those of existing
goldens (named in CASES), read from them rather than stored again; kp.npz holds the outputs only.  The AMP observation does
not depend on obs_v, so it is not repeated either: the source golden has it for the same inputs.

  A, B   envstep.npz inputs A / B (frame-grid times; blended times + global offset)
  C      envstep.npz inputs A with upright=False, local_root_obs=False (remove_base_rot before the heading)
  fut    fut.npz: fut_tracks with 3 samples ([B, T, 9K] -> [B, 9KT])
  getup  getup.npz: zero_out_far + cycle_motion, envs beyond close_distance and beyond far_distance (:834-845)
  occl   vr.npz occlusion G on the full body: position replaced, reference velocity kept (:847-851)
  vr     vr.npz: env_vr.yaml's Head + both hands tracked, reward over the subset

  python tests/golden/make_golden_kp.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import build_ref_env, run_ref_step, save, syn  # noqa: E402  (imports the reference through its shim)

# case -> (source golden, prefix of its input arrays, prefix of its v6 outputs for the same inputs)
CASES = {"A": ("envstep.npz", "A_in_", "A_out_"), "B": ("envstep.npz", "B_in_", "B_out_"), "C": ("envstep.npz", "A_in_", "C_out_"),
         "fut": ("fut.npz", "in_", "out_"), "getup": ("getup.npz", "in_", "out_"), "occl": ("vr.npz", "in_", "G_out_"),
         "vr": ("vr.npz", "in_", "E_out_")}
KEEP = ("obs", "rew", "reward_raw", "reset", "terminate", "ref_body_pos", "ref_body_rot", "ref_body_vel")


def source(case):
    name, pin, _ = CASES[case]
    z = np.load(os.path.join(HERE, name))
    g = {k: torch.from_numpy(z[k]) for k in z.files}
    m = syn.MotionData(**{k: g["tab_" + k] for k in syn.MotionData.__dataclass_fields__})
    st = syn.EnvState(**{k: g[pin + k].clone() for k in syn.EnvState.__dataclass_fields__})
    return g, m, st


def kp_env(env, K=None, T=1):
    """obs_v 7 with an observation buffer of the v7 width (9 K T task columns)."""
    J = env.num_bodies
    K = J if K is None else K
    env.obs_v = 7
    env.obs_buf = torch.zeros(env.num_envs, 1 + J * 15 - 3 + 9 * K * T)
    return env


def gen_kp():
    d = {}

    def put(tag, out):
        for k in KEEP:
            d[f"{tag}_out_{k}"] = out[k]

    for tag, kw in (("A", {}), ("B", {}), ("C", dict(upright=False, local_root_obs=False))):
        _, m, st = source(tag)
        put(tag, run_ref_step(kp_env(build_ref_env(m, st, **kw))))

    _, m, st = source("fut")
    env = build_ref_env(m, st)
    env._fut_tracks, env._num_traj_samples, env._traj_sample_timestep = True, 3, 1 / 10
    put("fut", run_ref_step(kp_env(env, T=3)))

    # getup: make_golden.gen_getup's steps with obs_v 7
    g, m, st = source("getup")
    N = st.body_state.shape[0]
    env = kp_env(build_ref_env(m, st))
    env.zero_out_far, env.zero_out_far_train, env.cycle_motion, env.cycle_motion_xp = True, False, True, False
    env.close_distance, env.far_distance = 0.25, 3
    env.max_episode_length = 15
    env._cycle_counter = torch.clamp_min(g["in_cycle_counter"] - 1, 0)       # pre_physics_step ran _update_cycle_count (:1076-1079)
    env._point_goal = g["in_point_goal"].clone()
    env._humanoid_root_states = env._rigid_body_state_reshaped[:, 0, :]
    env._motion_lib._device = torch.device("cpu")
    wrap = g["in_wrap"]
    torch.manual_seed(77)                 # the numbers sample_time_interval draws for the wrapping envs: in_cycle_phase
    phase = torch.zeros(N)
    phase[wrap] = torch.rand(int(wrap.sum()))
    assert torch.equal(phase, g["in_cycle_phase"])
    env._compute_reward(None)
    torch.manual_seed(77)
    env._compute_reset()
    env._compute_observations()
    put("getup", dict(obs=env.obs_buf, rew=env.rew_buf, reward_raw=env.reward_raw, reset=env.reset_buf, terminate=env._terminate_buf,
                      ref_body_pos=env.ref_body_pos, ref_body_rot=env.ref_body_rot, ref_body_vel=env.ref_body_vel))
    for k in ("start_times", "start_offsets", "global_offset", "cycle_counter", "point_goal"):
        d[f"getup_out_{k}"] = getattr(env, {"start_times": "_motion_start_times", "start_offsets": "_motion_start_times_offset"}.get(k, "_" + k))
    dist = torch.norm(st.body_state[:, 0, :3] - env.ref_body_pos[:, 0], dim=-1)
    print("kp getup: wrapping envs", int(wrap.sum()), "beyond close", int((dist > 0.25).sum()), "beyond far", int((dist > 3).sum()))

    g, m, st = source("occl")
    env = kp_env(build_ref_env(m, st))
    env._occl_training = True
    env.random_occlu_idx = g["G_occlusion"].clone()
    put("occl", run_ref_step(env))

    track = g["track"].tolist()
    env = kp_env(build_ref_env(m, st), K=len(track))
    env._track_bodies_id = torch.tensor(track)
    env._reset_bodies_id = torch.tensor(track)
    env._full_body_reward = False
    env.ref_body_pos_subset = torch.zeros(st.body_state.shape[0], len(track), 3)
    put("vr", run_ref_step(env))
    save("kp.npz", d)


if __name__ == "__main__":
    gen_kp()
