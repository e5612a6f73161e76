"""IMAmpAgent: the imitation agent of the reference (phc/learning/im_amp.py) on top of the phc_b200 AMPAgent.

The reference class adds three things to AMPAgent: `get_action` (deterministic / sampled action for evaluation), the evaluation
sweep `eval()` over the whole motion dataset with its per-step bookkeeping `_post_step_eval` (success rate, mean per-joint position
error over the un-terminated part of every clip, the failed / successful clip keys) and `update_training_data` (Auto-PMCP: the
failed clips re-weight the motion sampling).  This mirror keeps those method names and the returned dictionaries.

What is different: the bookkeeping lives on the device.  The reference stacks `info['mpjpe']` / `body_pos` / `body_pos_gt` of every
step in Python lists ([steps, N, J, 3] copied to the host), slices them per clip afterwards, and synchronises five to six times per
step (`.sum() > 0`, `.nonzero()`, `.max()`, `.item()`).  Here a step launches phc_eval_metrics_step, which adds the frame's errors to
per-env fp64 sums and frame counts (the per-step part of smpl_sim's `compute_metrics_lite`: global, root-relative and
Procrustes-aligned MPJPE, velocity and acceleration error), folds the termination flags, and reads back ONE packed scalar pair (the
step bound of the batch, the number of terminated envs).  At the end of the sweep the per-clip rows are reduced on the device in fp64
and read back once.  By default `eval()` returns the three keys `eval/success_rate`, `eval/mpjpe_all`, `eval/mpjpe_succ`, the MPJPEs
being means of per-clip means (every clip weighs the same).  With the agent config key `full_eval_metrics: True` it returns the
reference's eight keys with the reference's definitions: means over the frames of all (or of the successful) clips concatenated, so
long clips weigh more, `succ` falling back to `all` when no clip succeeded, NaN for a metric without frames.  Millimetres throughout.
"""
from __future__ import annotations

import glob
import os
from typing import Dict, List, Tuple

import numpy as np
import torch

from .. import ops
from .._lib import PHC_EVAL_ACC_FIELDS
from .amp_agent import AMPAgent


class IMAmpAgent(AMPAgent):
    def __init__(self, base_name, config):
        super().__init__(base_name, config)
        self.network_path = self.config.get("network_path", self.config.get("train_dir", "."))
        self.is_rnn, self.states, self.has_batch_dimension, self.clip_actions = False, None, True, bool(self.config.get("clip_actions", False))
        self.full_eval_metrics = bool(self.config.get("full_eval_metrics", False))

    # ---- im_amp.py:42-75 ------------------------------------------------------------------------------------------
    def get_action(self, obs_dict: Dict[str, torch.Tensor], is_determenistic: bool = False) -> torch.Tensor:
        res = self.get_action_values(obs_dict)
        a = res["mus"] if is_determenistic else res["actions"]
        return torch.clamp(a, -1.0, 1.0) if self.clip_actions else a

    def env_eval_step(self, env, actions):
        obs, rewards, dones, infos = env.step(actions)
        return obs, rewards, dones, infos

    # ---- im_amp.py:101-117 -----------------------------------------------------------------------------------------
    def restore(self, fn: str) -> None:
        """AMPAgent.restore, then the Auto-PMCP termination history of the newest `<network_path>/failed_*.pkl` (update_training_data
        writes one per evaluation) back into the motion sampling weights, so a resumed run keeps them."""
        super().restore(fn)
        fails = glob.glob(os.path.join(self.network_path, "failed_*"))
        if not fails:
            return
        newest = sorted(fails, key=lambda x: int(x.split("_")[-1].split(".")[0]))[-1]
        import joblib
        termination_history = joblib.load(newest)["termination_history"]
        ok = self.vec_env.env.task._motion_data.update_sampling_prob(termination_history)
        print(f"restored the termination history of {newest}" if ok else f"{newest}: termination history length does not match")

    # ---- im_amp.py:124-133 -----------------------------------------------------------------------------------------
    def update_training_data(self, failed_keys) -> None:
        task = self.vec_env.env.task
        lib = task._motion_data
        if getattr(task, "auto_pmcp", False):
            lib.update_hard_sampling_weight(failed_keys)
        elif getattr(task, "auto_pmcp_soft", False):
            lib.update_soft_sampling_weight(failed_keys)
        try:
            import joblib
            joblib.dump({"failed_keys": failed_keys, "termination_history": getattr(lib, "_termination_history", None)},
                        os.path.join(self.network_path, f"failed_{self.epoch_num:010d}.pkl"))
        except Exception:
            pass                                          # the dump is a convenience of the reference's training scripts

    # ---- im_amp.py:136-242 -----------------------------------------------------------------------------------------
    def eval(self) -> Dict[str, float]:
        """One sweep over the whole motion dataset, num_envs clips at a time, deterministic actions, UHC-style termination."""
        task = self.vec_env.env.task
        lib = task._motion_data
        if not hasattr(lib, "load_motions"):
            raise TypeError("IMAmpAgent.eval needs a loadable motion library (MotionLibSMPL): it walks the dataset in order")
        self.set_eval()
        N, dev = task.num_envs, self.device
        J = task._rigid_body_pos.shape[1]
        self.terminate_state = torch.zeros(N, dtype=torch.bool, device=dev)
        # per-env sums over the counted frames of the batch (phc_eval_metrics_step): mpjpe_g, mpjpe_l, mpjpe_pa, vel, accel [m], counts
        self._metric_acc = torch.zeros(N, PHC_EVAL_ACC_FIELDS, dtype=torch.float64, device=dev)
        self._metric_ring = torch.zeros(2, N, J, 3, device=dev)      # pred - gt of the last two steps
        self.terminate_memory: List[torch.Tensor] = []
        self._metric_rows: List[torch.Tensor] = []                    # per batch of clips: the [N, PHC_EVAL_ACC_FIELDS] sums
        self.curr_stpes, self.success_rate = 0, 0.0
        # the get-up schedule is off for the sweep (im_amp.py:167-172, :228-232)
        getup_probs = (task._recovery_episode_prob, task._fall_init_prob) if hasattr(task, "set_getup_probs") else None
        if getup_probs is not None:
            task.set_getup_probs(0, 0)
        task.set_eval_mode(True)
        task.begin_seq_motion_samples()
        try:
            done_mask = None
            info = {"end": False}
            while not info["end"]:
                obs = self.env_reset(done_mask)
                action = self.get_action(obs, is_determenistic=True)
                _, _, done, step_info = self.env_eval_step(self.vec_env.env, action)
                done_mask, info = self._post_step_eval(step_info, done.clone())
        finally:
            task.set_eval_mode(False)
            if getup_probs is not None:
                task.set_getup_probs(*getup_probs)
            if hasattr(lib, "load_motions"):
                task.resample_motions()                     # back to sampled training clips, every env reset (im_amp.py:226-238)
        self.update_training_data(info["failed_keys"])
        return info["eval_info"]

    def _post_step_eval(self, info, done) -> Tuple[torch.Tensor, Dict]:
        task = self.vec_env.env.task
        lib = task._motion_data
        num_unique = lib._num_unique_motions
        steps = lib.get_motion_num_steps().to(self.device)                      # [N] simulation steps of every loaded clip
        # a termination after the clip's last frame is not a failure (curr_step is one step behind the simulation)
        self.terminate_state |= (self.curr_stpes <= steps - 1) & (info["terminate"] != 0)
        # clips past the end of the dataset (the last batch wraps around) do not count
        ids = lib._curr_motion_ids.to(self.device)
        wrap = (ids == num_unique - 1).nonzero()
        counted = torch.ones_like(self.terminate_state) if wrap.numel() == 0 else (torch.arange(ids.shape[0], device=self.device) <= wrap[0, 0])
        alive = counted & ~self.terminate_state
        # this step's errors count for env e while it is inside its clip: the reference slices its lists [:num_steps - 1, e]
        ops.eval_metrics_step(info["body_pos"], info["body_pos_gt"], steps.int(), self.curr_stpes, self._metric_ring, self._metric_acc)
        # ONE read-back per step: the step bound of this batch and how many envs have terminated
        bound = torch.where(alive, steps, torch.zeros_like(steps)).max()
        packed = torch.stack((bound.float(), self.terminate_state.sum().float(), alive.any().float())).tolist()
        curr_max = int(packed[0]) if packed[2] else self.curr_stpes      # nobody left to wait for
        if self.curr_stpes >= curr_max:
            curr_max = self.curr_stpes + 1
        self.curr_stpes += 1
        end, eval_info, failed, succ = False, {}, [], []
        if self.curr_stpes >= curr_max or int(packed[1]) == task.num_envs:
            self.curr_stpes = 0
            self.terminate_memory.append(self.terminate_state.clone())
            self._metric_rows.append(self._metric_acc.clone())
            term = torch.cat(self.terminate_memory)[:num_unique]
            self.success_rate = float(1.0 - term.float().mean())
            if task.start_idx + task.num_envs >= num_unique:                   # the sweep is complete
                term_np = term.cpu().numpy()
                keys = np.asarray(lib._motion_data_keys)
                failed, succ = keys[term_np], keys[~term_np]
                rows = torch.cat(self._metric_rows)[:num_unique]
                if self.full_eval_metrics:
                    eval_info = self._full_metrics(rows, term, bool((~term_np).any()))
                else:
                    per_clip = rows[:, 0] / rows[:, 5].clamp(min=1.0)          # every clip's mean MPJPE, clips weighted equally
                    m_all = float(per_clip.mean()) * 1000.0
                    m_succ = float(per_clip[~term].mean()) * 1000.0 if bool((~term).any()) else m_all
                    eval_info = {"eval/success_rate": self.success_rate, "eval/mpjpe_all": m_all, "eval/mpjpe_succ": m_succ}
                end = True
            else:
                done[:] = 1                                                    # reset everything for the next batch of clips
                task.forward_motion_samples()
                self.terminate_state.zero_()
                self._metric_acc.zero_()
        return done, {"end": end, "eval_info": eval_info, "failed_keys": failed, "success_keys": succ}

    def _full_metrics(self, rows: torch.Tensor, term: torch.Tensor, any_succ: bool) -> Dict[str, float]:
        """compute_metrics_lite over the concatenated clips, as _post_step_eval logs it (im_amp.py:314-349): frame-weighted means of
        the per-frame joint means, in millimetres, over all clips and over the successful ones.  `rows` [num_unique, 8] fp64."""
        zero = torch.zeros((), dtype=rows.dtype, device=rows.device)
        sums = torch.stack((rows.sum(0), torch.where(term[:, None], zero, rows).sum(0)))        # [2, 8]: all, succ
        # metric / its frame count (0 / 0 = NaN, numpy's mean of nothing): mpjpe_g, mpjpe_l, mpjpe_pa over frames, vel, accel
        means = (sums[:, :5] / sums[:, [5, 5, 5, 6, 7]] * 1000.0).tolist()                         # the one read-back
        g, l, pa, vel, accel = means[1] if any_succ else means[0]
        return {"eval/success_rate": self.success_rate, "eval/mpjpe_all": means[0][0], "eval/mpjpe_succ": g, "eval/accel_dist": accel,
                "eval/vel_dist": vel, "eval/mpjpel_all": means[0][1], "eval/mpjpel_succ": l, "eval/mpjpe_pa": pa}
