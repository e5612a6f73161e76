"""Oracle of the keypoint-only task observation (env.obs_v: 7) in the same PyTorch terms as oracle/phc_oracle.py, whose
functions it reuses (test infrastructure).

  task_obs_v7        compute_imitation_observations_v7 (phc/env/tasks/humanoid_im.py:1362-1393)
  env_step_kp        oracle.env_step with the v7 task observation; occlusion overwrites the reference POSITION only (:847-851)
  env_step_getup_kp  oracle.env_step_getup with the v7 task observation; zero_out_far overwrites the positions of bodies 1.. and
                     every velocity, and turns a very far root target into a direction (:834-845)

Reward, reset, AMP observation and the ref_* buffers are those of v6 (the observation version changes none of them), so both
step functions take them from the v6 oracle and replace the task-observation columns."""
from typing import Dict, Optional

import torch
from torch import Tensor

from oracle import phc_oracle as O


def task_obs_v7(root_pos: Tensor, root_rot: Tensor, body_pos: Tensor, body_vel: Tensor, ref_pos: Tensor, ref_vel: Tensor,
                time_steps: int = 1, upright: bool = True) -> Tensor:
    """sim [N,K,3]; ref [N*T,K,3] (env-major, T samples per env) -> [N, T*K*9] = per sample [diff_pos | diff_vel | ref_pos - root]."""
    N, K, _ = body_pos.shape
    T = time_steps
    if not upright:
        root_rot = O.strip_base_rot(root_rot)
    hinv = O.heading_q(root_rot, inverse=True).view(N, 1, 1, 4)
    rp, rv = ref_pos.view(N, T, K, 3), ref_vel.view(N, T, K, 3)
    d_pos = O.qrot(hinv, rp - body_pos.view(N, 1, K, 3))
    d_vel = O.qrot(hinv, rv - body_vel.view(N, 1, K, 3))
    l_pos = O.qrot(hinv, rp - root_pos.view(N, 1, 1, 3))
    return torch.cat([x.reshape(N, T, -1) for x in (d_pos, d_vel, l_pos)], dim=-1).reshape(N, -1)


def _with_v7(out: Dict[str, Tensor], task: Tensor, v6_width: int) -> Dict[str, Tensor]:
    out["obs"] = torch.cat((out["obs"][:, :out["obs"].shape[1] - v6_width], task), dim=-1)
    return out


def env_step_kp(tab: O.MotionTables, cfg: O.StepConfig, body_state: Tensor, dof_state: Tensor, dof_force: Tensor,
                progress: Tensor, motion_ids: Tensor, start_times: Tensor, start_offsets: Tensor, global_offset: Tensor,
                amp_hist: Tensor, occlusion: Optional[Tensor] = None, shape_params: Optional[Tensor] = None,
                limb_weights: Optional[Tensor] = None) -> Dict[str, Tensor]:
    out = O.env_step(tab, cfg, body_state, dof_state, dof_force, progress, motion_ids, start_times, start_offsets, global_offset,
                     amp_hist, occlusion, shape_params, limb_weights)
    N, J, _ = body_state.shape
    bp, br, bv = body_state[..., 0:3], body_state[..., 3:7], body_state[..., 7:10]
    T = cfg.time_steps
    t_next = ((progress[:, None] + 1) * cfg.dt + torch.arange(T)[None, :] * cfg.traj_dt
              + start_times[:, None] + start_offsets[:, None]).flatten()
    refn = O.motion_state(tab, motion_ids.repeat_interleave(T), t_next, global_offset.repeat_interleave(T, dim=0))
    tb = list(range(J)) if cfg.track_bodies is None else cfg.track_bodies
    r_pos, r_vel = refn["rg_pos"][:, tb].clone(), refn["body_vel"][:, tb].clone()
    if occlusion is not None:
        assert T == 1
        oc = occlusion.bool()
        r_pos[oc] = bp[:, tb][oc]
    to = task_obs_v7(bp[:, 0], br[:, 0], bp[:, tb], bv[:, tb], r_pos, r_vel, T, cfg.upright)
    return _with_v7(out, to, 24 * len(tb) * T)


def env_step_getup_kp(tab: O.MotionTables, cfg: O.StepConfig, body_state: Tensor, dof_state: Tensor, dof_force: Tensor,
                      progress: Tensor, motion_ids: Tensor, start_times: Tensor, start_offsets: Tensor, global_offset: Tensor,
                      amp_hist: Tensor, point_goal: Tensor, cycle_counter: Tensor, cycle_phase: Tensor, zero_out_far: bool = True,
                      cycle_motion: bool = True, close_distance: float = 0.25, far_distance: float = 3.0,
                      max_episode_length: int = 300) -> Dict[str, Tensor]:
    out = O.env_step_getup(tab, cfg, body_state, dof_state, dof_force, progress, motion_ids, start_times, start_offsets, global_offset,
                           amp_hist, point_goal, cycle_counter, cycle_phase, zero_out_far, cycle_motion, close_distance, far_distance,
                           max_episode_length)
    N, J, _ = body_state.shape
    bp, br, bv = body_state[..., 0:3], body_state[..., 3:7], body_state[..., 7:10]
    # the observation follows the clip position after a wrap-around: the re-based bookkeeping env_step_getup returns
    t_next = (progress + 1) * cfg.dt + out["start_times"] + out["start_offsets"]
    refn = O.motion_state(tab, motion_ids, t_next, out["global_offset"])
    rp, rv = refn["rg_pos"].clone(), refn["body_vel"].clone()
    if zero_out_far:
        distance = torch.norm(bp[:, 0] - rp[:, 0], dim=-1)
        z = distance > close_distance
        rp[z, 1:] = bp[z, 1:]
        rv[z] = bv[z]
        vz = distance > far_distance
        rp[vz, 0] = ((rp[vz, 0] - bp[vz, 0]) / distance[vz, None] * far_distance) + bp[vz, 0]
    to = task_obs_v7(bp[:, 0], br[:, 0], bp, bv, rp, rv, 1, cfg.upright)
    return _with_v7(out, to, 24 * J)
