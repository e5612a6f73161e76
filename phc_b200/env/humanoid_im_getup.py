"""HumanoidImGetup / HumanoidImMCPGetup: the get-up schedule (phc/env/tasks/humanoid_im_getup.py, humanoid_im_mcp_getup.py) of
env_im_getup_mcp.yaml, env_im_x_getup_mcp.yaml and env_im_x_pnn.yaml on the phc_b200 kernels.

What the reference adds to HumanoidIm, and where it runs here:
  * recovery episodes: a terminated env may, with probability `recoveryEpisodeProb`, keep its state and get `recoverySteps` steps to
    get up; while its `_recovery_counter` runs it neither resets nor advances its progress (:135-146, :198-210) -- inside the fused
    step launch (PHC_FLAG_RECOVERY);
  * fall starts: other resetting envs start, with probability `fallInitProb`, from a state of a bank of fallen poses generated once by
    the simulator backend (:82-125, :168-182) -- phc_getup_reset selects them on the device, without a host sync;
  * their AMP history: every slot = the AMP vector of the current state for fall starts, the newest slot for recovery envs
    (humanoid_amp.py:559-573, :190-196) -- the observation-only launch with PHC_FLAG_AMP_CURRENT plus phc_amp_ring_fill;
  * the schedule (:67-74): before `getup_udpate_epoch` every reset is a fall start and no episode recovers; AMPAgent.pre_epoch applies it
    together with the reward weights (amp_agent.py:518-525).
flags.server_mode is not mirrored.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from .. import _lib, ops
from ..ops import _stream
from .humanoid_im import HumanoidIm
from .humanoid_im_mcp import HumanoidImMCP


class HumanoidImGetup(HumanoidIm):

    def __init__(self, cfg: Dict, sim_params=None, physics_engine=None, device_type: str = "cuda", device_id: int = 0,
                 headless: bool = True):
        self._getup_setup_probs(cfg)
        super().__init__(cfg, sim_params, physics_engine, device_type, device_id, headless)
        self._getup_setup_buffers()

    # ---- construction (humanoid_im_getup.py:44-65) ----------------------------------------------------------------
    def _getup_setup_probs(self, cfg: Dict) -> None:
        env = cfg["env"] if "env" in cfg else cfg
        self._recovery_episode_prob_tgt = self._recovery_episode_prob = float(env["recoveryEpisodeProb"])
        self._recovery_steps_tgt = self._recovery_steps = int(env["recoverySteps"])
        self._fall_init_prob_tgt = self._fall_init_prob = float(env["fallInitProb"])
        self.getup_udpate_epoch = int(env.get("getup_udpate_epoch", 10000))
        self._getup_schedule_cfg = bool(env.get("getup_schedule", False))     # humanoid.py:289

    def _getup_setup_buffers(self) -> None:
        if self._fut_tracks or self.num_extend_bodies > 0 or self._motion_lib.num_dofs > 0:
            raise NotImplementedError("the get-up schedule is built for time_steps 1 and spherical-joint humanoids without extend bodies "
                                      "(fut_tracks / hinge-joint robots are not supported)")
        if not hasattr(self.sim, "generate_fall_states"):
            raise TypeError("simulator backend lacks generate_fall_states() -> (root_states [N, 13], dof_pos [N, D]): HumanoidImGetup starts "
                            "episodes from a bank of fallen states the simulator generates (humanoid_im_getup.py:82-125; INTEGRATION.md, "
                            "'Simulator backend')")
        self.getup_schedule = self._getup_schedule_cfg
        N, dev = self.num_envs, self.device
        self.availalbe_fall_states = torch.zeros(N, dtype=torch.int64, device=dev)
        self.fall_id_assignments = torch.zeros(N, dtype=torch.int64, device=dev)
        self._recovery_counter = torch.zeros(N, dtype=torch.int32, device=dev)
        # the probabilities live on the device too: a graph-captured rollout reads them there, so schedule changes reach it
        self._p_dev = torch.zeros(2, dtype=torch.float32, device=dev)
        self.set_getup_probs(self._recovery_episode_prob, self._fall_init_prob)
        self._ref_init_mask = torch.zeros(N, dtype=torch.int64, device=dev)
        self._fall_mask = torch.zeros(N, dtype=torch.int64, device=dev)
        self._getup_u = torch.zeros(2, N, dtype=torch.float32, device=dev)
        self._plan.set_recovery_counter(self._recovery_counter)
        # the reset path's observation-only launch, which also writes the AMP vector of the current simulator state (newest slot)
        common = dict(cfg=self.step_cfg, mlib=self._motion_lib, body_state=self._rigid_body_state_reshaped, dof_state=self._dof_state,
                      dof_force=self.dof_force_tensor, progress=self.progress_buf, motion_ids=self._sampled_motion_ids,
                      start_times=self._motion_start_times, start_offsets=self._motion_start_times_offset, global_offset=self._global_offset,
                      point_goal=self._point_goal, cycle_phase=self._cycle_phase, occlusion=self.random_occlu_idx,
                      shape_params=self._plan._keep.get("shape_params"), limb_weights=self._plan._keep.get("limb_weights"))
        self._plan_reset_obs_getup = ops.EnvStepPlan(obs=self.obs_buf, only_where=self._reset_mask, obs_only=True, amp_obs_buf=self._amp_store,
                                                     amp_ring=self._amp_use_ring, ring_head_dev=self._ring_head, amp_current=True,
                                                     ref_cache=self._ref_cache, cycle_counter=self._cycle_counter, **common)
        self._generate_fall_states()

    def set_getup_probs(self, recovery_episode_prob: float, fall_init_prob: float) -> None:
        """Set `_recovery_episode_prob` / `_fall_init_prob` and the device copy phc_getup_reset reads (two fills on the stream, no sync),
        so that a graph-captured rollout sees the change.  A plain assignment to the two attributes (the reference's IMAmpAgent.eval
        does that, im_amp.py:167-172) is picked up by the next eagerly run reset()."""
        self._recovery_episode_prob, self._fall_init_prob = float(recovery_episode_prob), float(fall_init_prob)
        self._p_dev[0].fill_(self._recovery_episode_prob)
        self._p_dev[1].fill_(self._fall_init_prob)
        self._p_on_device = (self._recovery_episode_prob, self._fall_init_prob)

    def _generate_fall_states(self) -> None:
        """humanoid_im_getup.py:82-125: the backend simulates the bank (one fallen state per env); velocities zeroed, marks cleared."""
        root, dof_pos = self.sim.generate_fall_states()
        N, D = self.num_envs, self.num_dof
        root = torch.as_tensor(root).to(self.device, torch.float32).reshape(N, 13).clone()
        root[:, 7:13] = 0
        self._fall_root_states = root.contiguous()
        self._fall_dof_pos = torch.as_tensor(dof_pos).to(self.device, torch.float32).reshape(N, D).contiguous()
        self._fall_dof_vel = torch.zeros_like(self._fall_dof_pos)
        self.availalbe_fall_states.zero_()
        self.fall_id_assignments.zero_()

    # ---- schedule (:67-74) ----------------------------------------------------------------------------------------
    def update_getup_schedule(self, epoch_num: int, getup_udpate_epoch: int = 5000) -> None:
        if epoch_num > getup_udpate_epoch:
            self.set_getup_probs(self._recovery_episode_prob_tgt, self._fall_init_prob_tgt)
        else:
            self.set_getup_probs(0, 1)

    # ---- reset (:135-196 with humanoid.py:585-621, humanoid_amp.py:559-573) -----------------------------------------
    def reset(self, env_ids=None) -> torch.Tensor:
        """Reset of the envs selected by `env_ids` (None = all, a [N] mask, or indices): recovery / fall / reference-state starts chosen
        on the device (phc_getup_reset), reference-state init for the last group only, then the simulator push, observations and AMP
        history of every reset env."""
        self._set_mask(env_ids)
        if (self._recovery_episode_prob, self._fall_init_prob) != self._p_on_device:     # assigned directly since the last push
            self.set_getup_probs(self._recovery_episode_prob, self._fall_init_prob)
        lib, ml, st, N = self._lib, self._motion_lib, _stream(), self.num_envs
        self._getup_u.uniform_()                                   # bernoulli(p) == (u < p) for the recovery and the fall draw
        perm = torch.argsort(torch.rand(N, device=self.device))    # uniform permutation of the bank: the law of randperm
        ops.getup_reset(self._reset_mask, self._terminate_buf, self._getup_u[0], self._getup_u[1], perm, self._p_dev[0:1], self._p_dev[1:2],
                        self._recovery_steps, self._fall_root_states, self._fall_dof_pos, self.availalbe_fall_states, self.fall_id_assignments,
                        self._recovery_counter, self._rigid_body_state_reshaped, self._dof_state, self.progress_buf, self.reset_buf,
                        self._terminate_buf, self._ref_init_mask, self._fall_mask)
        # reference-state init (HumanoidIm.reset's launches) for the remaining envs only
        phase = torch.rand(N, device=self.device)
        if getattr(self, "_eval_mode", False) or bool(self.cfg.get("test", False)):
            phase.zero_()
        _lib.check(lib.phc_reset_bookkeeping(self._ref_init_mask.data_ptr(), phase.data_ptr(), self._plan._env_motion.data_ptr(), N,
                                             self._motion_start_times.data_ptr(), self._motion_start_times_offset.data_ptr(),
                                             self._global_offset.data_ptr(), self._cycle_counter.data_ptr(), self.progress_buf.data_ptr(),
                                             self.reset_buf.data_ptr(), self._terminate_buf.data_ptr(), st), "phc_reset_bookkeeping")
        _lib.check(lib.phc_set_env_state(C.byref(ml.c), self._sampled_motion_ids.data_ptr(), self._motion_start_times.data_ptr(),
                                         self._global_offset.data_ptr(), self._ref_init_mask.data_ptr(), N,
                                         self._rigid_body_state_reshaped.data_ptr(), self.sim.bodies_per_env,
                                         self._dof_state.data_ptr(), st), "phc_set_env_state")
        # _reset_env_tensors: every reset env's root / dof state goes to the simulation (recovery envs push their own)
        self.sim.set_env_state(self._reset_mask, self._rigid_body_state_reshaped, self._dof_state)
        # _compute_observations(env_ids) + _compute_amp_observations(env_ids): the newest AMP slot of every reset env
        self._plan_reset_obs_getup.run()
        # _init_amp_obs_ref for the reference-state starts (all slots), _init_amp_obs_default for the fall starts
        ops.amp_obs_demo(ml, self.step_cfg, self._sampled_motion_ids, self._motion_start_times, first_step=0,
                         num_steps=self._num_amp_obs_steps, out=self._amp_store, only_where=self._ref_init_mask,
                         slot_offset=0, slot_offset_dev=self._ring_head)
        ops.amp_ring_fill(self._amp_store, self._ring_head, self._fall_mask)
        return self.obs_buf

    def _reload_motions(self, random_sample: bool, start_idx: int = 0) -> None:
        super()._reload_motions(random_sample, start_idx)
        self._plan_reset_obs_getup.set_motion_lib(self._motion_lib)

    def resample_motions(self):
        """humanoid_im_getup.py:127-133: HumanoidIm's resample, a new fall-state bank (unless test), then a reset of every env."""
        super().resample_motions()
        if hasattr(self, "_plan_reset_obs_getup") and not hasattr(self._motion_data, "load_motions"):
            self._plan_reset_obs_getup.refresh_motion_params()
        if not bool(self.cfg.get("test", False)):
            self._generate_fall_states()
        self.reset()


class HumanoidImMCPGetup(HumanoidImGetup, HumanoidImMCP):
    """humanoid_im_mcp_getup.py:26-30: the composer task with the get-up schedule."""

    def __init__(self, cfg: Dict, sim_params=None, physics_engine=None, device_type: str = "cuda", device_id: int = 0,
                 headless: bool = True, pnn_checkpoint: Optional[Dict] = None):
        self._getup_setup_probs(cfg)
        HumanoidImMCP.__init__(self, cfg, sim_params, physics_engine, device_type, device_id, headless, pnn_checkpoint=pnn_checkpoint)
        self._getup_setup_buffers()
