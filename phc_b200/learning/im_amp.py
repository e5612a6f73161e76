"""IMAmpAgent: the imitation agent of the reference (phc/learning/im_amp.py) on top of the phc_b200 AMPAgent.

The reference class adds three things to AMPAgent: `get_action` (deterministic / sampled action for evaluation), the evaluation
sweep `eval()` over the whole motion dataset with its per-step bookkeeping `_post_step_eval` (success rate, mean per-joint position
error over the un-terminated part of every clip, the failed / successful clip keys) and `update_training_data` (Auto-PMCP: the
failed clips re-weight the motion sampling).  This mirror keeps those method names and the returned dictionaries.

What is different: the bookkeeping lives on the device.  The reference stacks `info['mpjpe']` / `body_pos` / `body_pos_gt` of every
step in Python lists ([steps, N, J, 3] copied to the host), slices them per clip afterwards, and synchronises five to six times per
step (`.sum() > 0`, `.nonzero()`, `.max()`, `.item()`).  Here a step adds the masked per-env error to two [N] accumulators and folds
the termination flags, and reads back ONE packed scalar pair (the step bound of the batch, the number of terminated envs).
`compute_metrics_lite` (smpl_sim, absent from the reference tree: acceleration / velocity / Procrustes-aligned errors) is not restated;
`eval/mpjpe_all` and `eval/mpjpe_succ` are the global MPJPE the reference logs under those keys, in millimetres like `mpjpe_g`.
"""
from __future__ import annotations

import os
from typing import Dict, List, Tuple

import numpy as np
import torch

from .amp_agent import AMPAgent


class IMAmpAgent(AMPAgent):
    def __init__(self, base_name, config):
        super().__init__(base_name, config)
        self.network_path = self.config.get("network_path", self.config.get("train_dir", "."))
        self.is_rnn, self.states, self.has_batch_dimension, self.clip_actions = False, None, True, bool(self.config.get("clip_actions", False))

    # ---- im_amp.py:42-75 ------------------------------------------------------------------------------------------
    def get_action(self, obs_dict: Dict[str, torch.Tensor], is_determenistic: bool = False) -> torch.Tensor:
        res = self.get_action_values(obs_dict)
        a = res["mus"] if is_determenistic else res["actions"]
        return torch.clamp(a, -1.0, 1.0) if self.clip_actions else a

    def env_eval_step(self, env, actions):
        obs, rewards, dones, infos = env.step(actions)
        return obs, rewards, dones, infos

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
        self.terminate_state = torch.zeros(N, dtype=torch.bool, device=dev)
        self._err_sum = torch.zeros(N, device=dev)        # sum over the counted steps of the env's MPJPE
        self._err_cnt = torch.zeros(N, device=dev)
        self.terminate_memory: List[torch.Tensor] = []
        self.mpjpe_all: List[torch.Tensor] = []
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
        # this step's error counts for env e while it is inside its clip: the reference averages all_mpjpe[:num_steps - 1, e]
        inside = self.curr_stpes < (steps - 1)
        self._err_sum += torch.where(inside, info["mpjpe"], torch.zeros_like(self._err_sum))
        self._err_cnt += inside.float()
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
            self.mpjpe_all.append(self._err_sum / self._err_cnt.clamp(min=1.0))
            term = torch.cat(self.terminate_memory)[:num_unique]
            self.success_rate = float(1.0 - term.float().mean())
            if task.start_idx + task.num_envs >= num_unique:                   # the sweep is complete
                per_clip = torch.cat(self.mpjpe_all)[:num_unique]
                term_np = term.cpu().numpy()
                keys = np.asarray(lib._motion_data_keys)
                failed, succ = keys[term_np], keys[~term_np]
                m_all = float(per_clip.mean()) * 1000.0
                m_succ = float(per_clip[~term].mean()) * 1000.0 if bool((~term).any()) else m_all
                eval_info = {"eval/success_rate": self.success_rate, "eval/mpjpe_all": m_all, "eval/mpjpe_succ": m_succ}
                end = True
            else:
                done[:] = 1                                                    # reset everything for the next batch of clips
                task.forward_motion_samples()
                self.terminate_state.zero_()
                self._err_sum.zero_()
                self._err_cnt.zero_()
        return done, {"end": end, "eval_info": eval_info, "failed_keys": failed, "success_keys": succ}
