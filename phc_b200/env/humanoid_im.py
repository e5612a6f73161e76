"""HumanoidIm task on the phc_b200 kernels: same buffers, method names and step order as the reference task stack

    BaseTask -> Humanoid -> HumanoidAMP -> HumanoidAMPTask -> HumanoidIm
    (phc/env/tasks/{base_task,humanoid,humanoid_amp,humanoid_amp_task,humanoid_im}.py)

with the arithmetic of a whole post-physics step in ONE kernel launch (ops.EnvStepPlan -> phc_env_step) and the
episode-reset path expressed as per-env MASKS instead of `env_ids = dones.nonzero()` index lists, so a rollout step
needs no device->host synchronisation.

The rigid-body simulator is not part of this package.  `HumanoidIm` talks to it through a small backend object:
  * `SyntheticSim` (this file): seeded synthetic rigid-body state (bench, tests, smoke -- SURVEY.md section 8d);
  * an Isaac Gym backend has to expose the same tensors (`rigid_body_state [N, bodies_per_env, 13]`,
    `dof_state [N, D, 2]`, `dof_force [N, D]`, Humanoid._setup_tensors humanoid.py:179-247) and `simulate(actions)`
    = pre_physics_step + gym.simulate + refresh (humanoid.py:1522-1619, humanoid_amp.py:639-660); INTEGRATION.md.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence

import torch

from collections.abc import Mapping

from .. import _lib, ops, synthetic as syn
from ..ops import _ptr, _stream
from . import backends


class _Extras(dict):
    """`extras` of the task with the reference's `amp_obs` entry (humanoid_amp.py:207-208: the flattened newest-first AMP window,
    [N, S*A]) materialised from the ring only when somebody reads it; phc_b200's own agent takes `amp_obs_export` instead and has the
    window written straight into its experience buffer."""

    def __init__(self, task):
        super().__init__()
        self._task = task

    def __getitem__(self, k):
        if k == "amp_obs" and not dict.__contains__(self, k):
            t = self._task
            return t._amp_obs_buf.view(t.num_envs, -1)
        return super().__getitem__(k)

    def __contains__(self, k):
        return k == "amp_obs" or super().__contains__(k)

    def get(self, k, default=None):
        return self[k] if k in self else default


class SyntheticSim:
    """Stand-in for the simulator: a bank of K seeded rigid-body snapshots that `simulate()` cycles through.
    With `host_bank=True` the bank lives in pinned host memory and every step pays the host->device copy (the
    end-to-end measurement of bench.py); otherwise snapshots are device resident."""

    graph_safe = True      # simulate() only enqueues copies on the current stream: a rollout over this backend can be a CUDA graph
                           # (bank size 4 divides the rollout lengths in use, so every rollout sees the same snapshot sequence)

    def __init__(self, motion: syn.MotionData, num_envs: int, device, seed: int = 0, bank: int = 4, host_bank: bool = False,
                 amp_dim: int = 196, amp_steps: int = 10):
        self.device = torch.device(device)
        self.num_envs = num_envs
        make = syn.make_robot_env_state if isinstance(motion, syn.RobotMotionData) else syn.make_env_state
        states = [make(motion, num_envs, seed=seed * 100 + k, amp_dim=amp_dim, amp_steps=amp_steps) for k in range(bank)]
        self.init_state = states[0]
        keep = lambda ts: torch.stack(ts).pin_memory() if host_bank else torch.stack(ts).to(self.device)
        self._body = keep([s.body_state for s in states])
        self._dof = keep([s.dof_state for s in states])
        self._force = keep([s.dof_force for s in states])
        self.rigid_body_state = states[0].body_state.to(self.device).clone()
        self.dof_state = states[0].dof_state.to(self.device).clone()
        self.dof_force = states[0].dof_force.to(self.device).clone()
        self.bodies_per_env = self.rigid_body_state.shape[1]
        self._k = 0
        self.h2d_bytes_per_step = (self.rigid_body_state.numel() + self.dof_state.numel() + self.dof_force.numel()) * 4 if host_bank else 0

    def set_env_state(self, mask: torch.Tensor, rigid_body_state: torch.Tensor, dof_state: torch.Tensor) -> None:
        """Backend hook of HumanoidIm.reset (Humanoid._reset_env_tensors, humanoid.py:590-621): apply the state HumanoidIm wrote
        into the rows of `rigid_body_state` / `dof_state` flagged by `mask` to the simulation.  The synthetic stand-in has no
        dynamics to reset -- its next snapshot replaces every row anyway -- so there is nothing to do."""
        return

    def generate_fall_states(self, seed: int = 0):
        """Backend hook of HumanoidImGetup (humanoid_im_getup.py:82-125): a bank of one "fallen" state per env, (root_states [N, 13],
        dof_pos [N, D]).  The stand-in has no physics to let the characters fall, so the bank is the first snapshot with a seeded random
        unit root rotation (the reference's randn + normalize, :90-91) and zero root velocities; deterministic for a given seed."""
        g = torch.Generator().manual_seed(int(seed))
        root = self.init_state.body_state[:, 0, :].detach().cpu().clone().float()
        q = torch.randn(root.shape[0], 4, generator=g)
        root[:, 3:7] = torch.nn.functional.normalize(q, dim=-1)
        root[:, 7:13] = 0
        dof_pos = self.init_state.dof_state[..., 0].detach().cpu().clone().float()
        return root.to(self.device), dof_pos.to(self.device)

    def simulate(self, actions: Optional[torch.Tensor]) -> None:
        k = self._k = (self._k + 1) % self._body.shape[0]
        self.rigid_body_state.copy_(self._body[k], non_blocking=True)
        self.dof_state.copy_(self._dof[k], non_blocking=True)
        self.dof_force.copy_(self._force[k], non_blocking=True)


class HumanoidIm:
    """Imitation task.  cfg keys (all optional except the motion data): the `env` block of env_im.yaml plus
    `motion_data` (synthetic.MotionData or any object with the MotionLibBase table attributes) and `sim` (backend)."""

    def __init__(self, cfg: Dict, sim_params=None, physics_engine=None, device_type: str = "cuda", device_id: int = 0,
                 headless: bool = True):
        env = cfg.get("env", cfg)
        self.cfg = cfg
        robot_cfg = cfg.get("robot", {}) or {}

        def rcfg(key, default):       # robot-level switches: cfg.robot.<key> as run_hydra.py builds the tree (humanoid.py:285-330), else top level
            return robot_cfg.get(key, cfg.get(key, default)) if isinstance(robot_cfg, Mapping) else cfg.get(key, default)
        self._rcfg = rcfg
        self.device = torch.device(f"{device_type}:{device_id}" if device_type == "cuda" else device_type)
        torch.cuda.set_device(self.device)
        self.headless = headless
        self.num_envs = int(env.get("num_envs", 3072))
        # dt = control_freq_inv * sim_params.dt (humanoid.py:74-76); sim_params is Isaac Gym's object when the reference constructs us
        sim_block = cfg.get("sim", None)
        sim_dt = getattr(sim_params, "dt", None) or (sim_block.get("dt") if isinstance(sim_block, Mapping) else None) or cfg.get("sim_dt", 1.0 / 60.0)
        self.dt = float(env.get("controlFrequencyInv", 2)) * float(sim_dt)
        self.max_episode_length = int(env.get("episode_length", 300))
        self.humanoid_type = rcfg("humanoid_type", "smpl")
        self._num_amp_obs_steps = int(env.get("numAMPObsSteps", 10))
        self.power_reward = bool(env.get("power_reward", True))
        self.power_coefficient = float(env.get("power_coefficient", 0.0005))
        self._fut_tracks = bool(env.get("fut_tracks", False))
        self._num_traj_samples = int(env.get("numTrajSamples", 3)) if self._fut_tracks else 1
        self._traj_sample_timestep = 1.0 / float(env.get("trajSampleTimestepInv", 30)) if self._fut_tracks else 0.0
        self.shape_resampling_interval = int(env.get("shape_resampling_interval", 500))
        self.temp_running_mean = True
        self.getup_schedule = False
        self.kin_lr = False
        self.fitting = False
        self.has_task = True
        self.viewer = None
        # env_im_getup_mcp.yaml (humanoid.py:294-330): clip wrap-around and the far-reference handling, both inside the fused launch
        self.cycle_motion = bool(env.get("cycle_motion", False))
        self.cycle_motion_xp = bool(env.get("cycle_motion_xp", False))
        self.zero_out_far = bool(env.get("zero_out_far", False))
        self.zero_out_far_train = bool(env.get("zero_out_far_train", True)) and self.zero_out_far
        self.close_distance = float(env.get("close_distance", 0.25))
        self.far_distance = float(env.get("far_distance", 3))
        self._zero_out_far_steps = int(env.get("zero_out_far_steps", 90))
        self.max_episode_length = int(env.get("episode_length", 300))
        if self.cycle_motion_xp or self.zero_out_far_train:
            raise NotImplementedError("cycle_motion_xp / zero_out_far_train (random re-placement, humanoid_im.py:966-980, :1131-1140) "
                                      "are not on the fused path; the shipped getup config has both off")
        # env.obs_v (_compute_task_obs, humanoid_im.py:772-853): 6 for the shipped yamls, 7 for the keypoint models.  The default is 6
        # (every shipped yaml sets it) although the reference's own is 1 (humanoid.py:296)
        self.obs_v = int(env.get("obs_v", 6))
        if self.obs_v not in (6, 7):
            fn = {1: "compute_imitation_observations", 2: "compute_imitation_observations_v2", 3: "compute_imitation_observations_v3",
                  4: "compute_imitation_observations_v6 with the obs_v 4 size", 5: "compute_imitation_observations_v6 + one-hot motion types",
                  8: "compute_imitation_observations_v8", 9: "compute_imitation_observations_v9"}.get(self.obs_v, "no reference observation")
            raise NotImplementedError(f"env.obs_v {self.obs_v} ({fn}, humanoid_im.py) is not built; obs_v 6 and 7 (keypoints) are")

        # ---- simulator backend: explicit object, the synthetic stand-in for synthetic motion data, or the registered factory ----
        sim = cfg.get("sim_backend", None)
        if sim is None and sim_block is not None and not isinstance(sim_block, Mapping):
            sim = sim_block                           # round-1 spelling: the backend object under cfg["sim"] (the reference keeps physx settings there)
        synthetic_data = isinstance(cfg.get("motion_data", None), (syn.MotionData, syn.RobotMotionData))
        if sim is None and not synthetic_data:
            sim = backends.make_backend(cfg, sim_params, physics_engine, device_type, device_id, headless)
        # ---- motion library (tables as MotionLibBase keeps them) -> packed device format -----------------------
        m = cfg.get("motion_data", None)
        if m is None:
            m = self._load_motion(env, sim)           # Humanoid._load_motion (humanoid_im.py:300-360): MotionLibSMPL on env.motion_file
        self._motion_data = m
        d = m.to(self.device) if hasattr(m, "to") else m
        robot = hasattr(d, "gts_t")            # hinge-joint robot tables (phc/utils/motion_lib_real.py): h1 / g1
        if robot:
            dev = self.device
            self._motion_lib = ops.pack_robot_motion_lib(d.gts_t.to(dev), d.grs_t.to(dev), d.gvs_t.to(dev), d.gavs_t.to(dev),
                                                         d.dof_pos.to(dev), d.dvs.to(dev), d.num_bodies, d.lengths.to(dev),
                                                         d.num_frames.to(dev), d.dts.to(dev), d.length_starts.to(dev))
            if self.humanoid_type == "smpl":
                self.humanoid_type = "h1"
        elif isinstance(getattr(d, "packed", None), ops.PackedMotionLib):
            self._motion_lib = d.packed           # phc_b200.motion_lib.MotionLibSMPL: loaded and packed on the device already
        else:
            self._motion_lib = ops.pack_motion_lib(d.gts, d.grs, d.gvs, d.gavs, d.lrs, d.dvs, d.lengths, d.num_frames, d.dts,
                                                   d.length_starts)
        J = self._motion_lib.num_bodies
        self.num_bodies = J
        self.num_dof = self._motion_lib.dofs
        # cfg.robot.extend_config (humanoid_im.py:74-82): parent body index + position in the parent frame
        ext = rcfg("extend_config", [dict(parent=p, pos=q) for p, q in zip(syn.H1_EXT_PARENTS, syn.H1_EXT_POS)] if robot else [])
        body_names = rcfg("body_names", None) or getattr(sim, "body_names", None)        # the reference names parents (extend_config.parent_name)
        self.extend_body_parent_ids = [int(e["parent"]) if "parent" in e else list(body_names).index(e["parent_name"]) for e in ext]
        self.extend_body_pos_in_parent = [list(e["pos"]) for e in ext]
        self.num_extend_bodies = len(ext)
        key_bodies = env.get("key_body_ids", syn.H1_KEY_BODIES if robot else (syn.SMPL_KEY_BODIES if J == 24 else [J - 1]))
        reset_bodies = env.get("reset_body_ids", syn.SMPL_RESET_BODIES if (J == 24 and not robot) else None)
        dof_subset = env.get("dof_subset", syn.SMPL_DOF_SUBSET if (J == 24 and not robot and rcfg("has_dof_subset", True)) else None)
        # env.trackBodies / env.reset_bodies (names or ids; humanoid_im.py:64-66): the tracked subset of env_vr.yaml; reset bodies default
        # to the tracked ones.  env.full_body_reward False = the reward follows the subset (:926-935)
        names = list(rcfg("body_names", None) or getattr(sim, "body_names", None) or (syn.SMPL_BODY_NAMES if (J == 24 and not robot) else []))
        to_ids = lambda lst: [names.index(b) if isinstance(b, str) else int(b) for b in lst]
        track = env.get("trackBodies", None)
        self._track_bodies_id = None if track is None or len(track) in (0, J) else to_ids(track)
        tracked = self._track_bodies_id if self._track_bodies_id is not None else list(range(J))
        self._track_bodies = [names[b] for b in tracked] if names else tracked       # humanoid_im.py:64-66 keeps the names
        if "reset_bodies" in env:
            reset_bodies = to_ids(env["reset_bodies"])
        elif self._track_bodies_id is not None and "reset_body_ids" not in env:
            reset_bodies = list(self._track_bodies_id)
        self._full_body_reward = bool(env.get("full_body_reward", True))
        # _occl_training (:96-97, :797-804, :1081-1092): which tracked bodies are hidden from the policy this step
        self._occl_training = bool(env.get("occlusion_training", False))
        self._occl_training_prob = float(env.get("occlusion_training_prob", 0.1))
        self.random_occlu_idx = self.random_occlu_count = None
        if self._occl_training:
            if self._track_bodies_id is not None:
                raise NotImplementedError("occlusion_training with a tracked-body subset: the reference indexes random_occlu_idx by body id in the "
                                          "reset test (humanoid_im.py:1181), which only works with every body tracked")
            self.random_occlu_idx = torch.zeros(self.num_envs, J, dtype=torch.bool, device=self.device)
            self.random_occlu_count = torch.zeros(self.num_envs, J, dtype=torch.int64, device=self.device)
        # has_shape_obs / has_weight_obs (humanoid.py:271-274, :1469-1470): per-env body shape (gender + betas = humanoid_shapes[:, :-6] for the
        # SMPL family) and limb lengths / weights appended to the self observation; the simulator side owns both
        self._has_shape_obs, self._has_limb_weight_obs = bool(rcfg("has_shape_obs", False)), bool(rcfg("has_weight_obs", False))
        shape_params = limb_weights = None
        if self._has_shape_obs:
            hs = torch.as_tensor(sim.humanoid_shapes, dtype=torch.float32).to(self.device)
            shape_params = (hs[:, :-6] if self.humanoid_type in ("smpl", "smplh", "smplx") else hs).contiguous()
        if self._has_limb_weight_obs:
            limb_weights = torch.as_tensor(sim.humanoid_limb_and_weights, dtype=torch.float32).to(self.device).contiguous()
        self.step_cfg = ops.EnvStepConfig(
            dt=self.dt, time_steps=self._num_traj_samples, traj_dt=self._traj_sample_timestep,
            upright=bool(rcfg("has_upright_start", True)), local_root_obs=bool(env.get("local_root_obs", True)),
            root_height_obs=bool(env.get("root_height_obs", True)), power_reward=self.power_reward,
            power_coef=self.power_coefficient, early_term=bool(env.get("enableEarlyTermination", True)),
            key_bodies=key_bodies, reset_bodies=reset_bodies, term_dist=float(env.get("terminationDistance", 0.25)),
            dof_subset=dof_subset, amp_steps=self._num_amp_obs_steps, ext_parents=self.extend_body_parent_ids,
            ext_pos=self.extend_body_pos_in_parent, zero_out_far=self.zero_out_far, close_distance=self.close_distance,
            far_distance=self.far_distance, cycle_motion=self.cycle_motion, max_episode_length=self.max_episode_length,
            specialise=bool(cfg.get("specialised_step", True)), track_bodies=self._track_bodies_id, full_body_reward=self._full_body_reward,
            term_use_mean=bool(cfg.get("im_eval", False)) and not bool(env.get("strict_eval", False)),   # humanoid_im.py:1180
            obs_v=self.obs_v)
        self._key_body_ids, self._reset_bodies_id, self.dof_subset = key_bodies, reset_bodies, dof_subset

        # ---- simulator backend and its tensors (Humanoid._setup_tensors) ---------------------------------------
        self.sim = sim if sim is not None else SyntheticSim(m, self.num_envs, self.device, seed=int(cfg.get("seed", 0)),
                                                             host_bank=bool(cfg.get("host_sim_bank", False)),
                                                             amp_dim=13 + 2 * self.num_dof + 3 * len(key_bodies) if robot else 196)
        if not hasattr(self.sim, "set_env_state"):
            raise TypeError("simulator backend lacks set_env_state(mask, rigid_body_state, dof_state): without it an episode reset would only "
                            "rewrite observation-side tensors and the physics would keep running from the old state (INTEGRATION.md, "
                            "'Simulator backend')")
        self._rigid_body_state_reshaped = self.sim.rigid_body_state
        self._rigid_body_pos = self._rigid_body_state_reshaped[..., :J, 0:3]
        self._rigid_body_rot = self._rigid_body_state_reshaped[..., :J, 3:7]
        self._rigid_body_vel = self._rigid_body_state_reshaped[..., :J, 7:10]
        self._rigid_body_ang_vel = self._rigid_body_state_reshaped[..., :J, 10:13]
        self._dof_state = self.sim.dof_state
        self._dof_pos, self._dof_vel = self._dof_state[..., 0], self._dof_state[..., 1]
        self.dof_force_tensor = self.sim.dof_force

        # ---- task buffers (BaseTask buffers base_task.py:99-104 + HumanoidIm extras) ----------------------------
        N, dev = self.num_envs, self.device
        i64 = torch.int64
        self.progress_buf = torch.zeros(N, dtype=i64, device=dev)
        self._sampled_motion_ids = (torch.arange(N, device=dev) % self._motion_lib.num_motions).to(i64)
        self._motion_start_times = torch.zeros(N, device=dev)
        self._motion_start_times_offset = torch.zeros(N, device=dev)
        self._global_offset = torch.zeros(N, 3, device=dev)
        self._cycle_counter = torch.zeros(N, dtype=torch.int32, device=dev)
        self._reset_mask = torch.zeros(N, dtype=i64, device=dev)
        self._point_goal = torch.zeros(N, device=dev)                 # humanoid_im.py:95
        self._cycle_phase = torch.zeros(N, device=dev)                # uniform numbers for clips that wrap this step
        self.extras: Dict[str, torch.Tensor] = _Extras(self)

        common = dict(cfg=self.step_cfg, mlib=self._motion_lib, body_state=self._rigid_body_state_reshaped,
                      dof_state=self._dof_state, dof_force=self.dof_force_tensor, progress=self.progress_buf,
                      motion_ids=self._sampled_motion_ids, start_times=self._motion_start_times,
                      start_offsets=self._motion_start_times_offset, global_offset=self._global_offset,
                      point_goal=self._point_goal, cycle_phase=self._cycle_phase, occlusion=self.random_occlu_idx, shape_params=shape_params,
                      limb_weights=limb_weights)
        # AMP history: a RING [N, S, A] (one 784-byte slot written per step) instead of the reference's per-step shift of
        # the whole window (humanoid_amp.py:662-670); the newest-first window is exported on demand (`_amp_obs_buf`,
        # `export_amp_obs`).  amp_window_shift=True in cfg restores the in-kernel reference-style shift.
        self._amp_use_ring = not bool(cfg.get("amp_window_shift", False))
        # Interpolated reference pose kept across steps: the pose a launch blends for its observation (time t + dt) is the
        # pose the next launch needs for reward / reset (SURVEY.md 8d counts it that way).  Rows are 13-float body records;
        # ref_body_pos / rot / vel / ang_vel (humanoid_im.py:855-868) are strided views of it.  ref_pose_cache=False in cfg
        # re-interpolates every step and keeps separate ref_* buffers.
        self._use_ref_cache = bool(cfg.get("ref_pose_cache", True))
        J = self._motion_lib.num_bodies
        self._ref_cache = torch.zeros(N, int(self._motion_lib.frames_body.shape[1]), device=dev) if self._use_ref_cache else None
        # flags.im_eval (humanoid_im.py:674-680; also selects the mean-distance termination, :1180): extras['mpjpe'], body_pos(_gt)
        self.im_eval = bool(cfg.get("im_eval", False))
        # the ring head lives on the device: a rollout step then differs from the next in nothing the host passes
        self._ring_head = torch.zeros(1, dtype=torch.int32, device=dev) if self._amp_use_ring else None
        self._plan = ops.EnvStepPlan(cycle_counter=self._cycle_counter, with_ref_buffers=not self._use_ref_cache, ring_head_dev=self._ring_head,
                                     with_eval_extras=self.im_eval,
                                     amp_ring=self._amp_use_ring, ref_cache=self._ref_cache,
                                     reward_from_cache=self._use_ref_cache, **common)
        p = self._plan
        if self._use_ref_cache:
            rec = self._ref_cache[:, :13 * J].view(N, J, 13)
            p.ref_body_pos, p.ref_body_rot, p.ref_body_vel, p.ref_body_ang_vel = rec[..., 0:3], rec[..., 3:7], rec[..., 7:10], rec[..., 10:13]
        self.obs_buf, self.rew_buf, self.reward_raw = p.obs, p.rew, p.reward_raw
        self.reset_buf, self._terminate_buf = p.reset, p.terminate
        self._amp_store = p.amp_obs_buf                              # ring (or the shifted window itself)
        self._amp_window = torch.zeros_like(self._amp_store) if self._amp_use_ring else self._amp_store
        self.ref_body_pos, self.ref_body_rot, self.ref_body_vel = p.ref_body_pos, p.ref_body_rot, p.ref_body_vel
        self._num_amp_obs_per_step = p.amp_dim
        self._curr_amp_obs_buf = self._hist_amp_obs_buf = None        # reference views of the shifted window; not kept with the ring
        self.self_obs_buf = self.obs_buf[:, :p.self_dim]
        # observation-only re-computation for just-reset envs (_compute_observations(env_ids))
        self._plan_reset_obs = ops.EnvStepPlan(obs=self.obs_buf, only_where=self._reset_mask, obs_only=True, with_amp=False,
                                               ref_cache=self._ref_cache, cycle_counter=self._cycle_counter, **common)
        self._lib = _lib.load()
        self._kb = (C.c_int32 * len(key_bodies))(*[int(b) for b in key_bodies])
        self.actions = None
        if hasattr(self.sim, "pd_action_offset"):         # the backend knows the dof limits (Humanoid._build_pd_action_offset_scale)
            self.set_pd_action_map(self.sim.pd_action_offset, self.sim.pd_action_scale)

    # ---- sizes (Humanoid.get_obs_size & co) --------------------------------------------------------------------
    def get_obs_size(self):
        return self._plan.obs_dim

    def get_self_obs_size(self):
        return self._plan.self_dim

    def get_task_obs_size(self):
        return self._plan.task_dim

    def get_action_size(self):
        return self.num_dof

    def get_num_amp_obs(self):
        return self._num_amp_obs_steps * self._num_amp_obs_per_step

    def get_task_obs_size_detail(self):
        """humanoid_im.py:522-537: what the network builders read from the task."""
        env = self.cfg.get("env", self.cfg)
        return {"target": self._plan.task_dim, "fut_tracks": self._fut_tracks, "num_traj_samples": self._num_traj_samples, "obs_v": self.obs_v,
                "track_bodies": self._track_bodies, "models_path": env.get("models", []), "num_prim": env.get("num_prim", 2),
                "training_prim": env.get("training_prim", 1), "actors_to_load": env.get("actors_to_load", 2),
                "has_lateral": env.get("has_lateral", True)}

    def get_running_mean_size(self):
        return (self.get_obs_size(),)

    # ---- step ---------------------------------------------------------------------------------------------------
    def set_pd_action_map(self, offset: torch.Tensor, scale: torch.Tensor, action_idx=None, zero_dofs=()) -> None:
        """The affine action -> PD-target map of Humanoid._build_pd_action_offset_scale (humanoid.py:1331-1380; built from the
        asset's dof limits, so the backend supplies it): `_pd_action_offset`, `_pd_action_scale` [num_dof]; `action_idx` (reduce_action:
        the dofs the policy drives); `zero_dofs`: dof indices frozen at 0 (_freeze_hand / _freeze_toe).  Once set, step() turns the
        policy output into PD targets on the device (phc_pd_targets) before it reaches the backend's simulate()."""
        D = self.num_dof
        self._pd_action_offset = offset.to(self.device, torch.float32).contiguous()
        self._pd_action_scale = scale.to(self.device, torch.float32).contiguous()
        assert self._pd_action_offset.shape == (D,) and self._pd_action_scale.shape == (D,)
        self._pd_dof_of_action = None
        if action_idx is not None:
            m = torch.full((D,), -1, dtype=torch.int32)
            m[torch.as_tensor(action_idx, dtype=torch.long)] = torch.arange(len(action_idx), dtype=torch.int32)
            self._pd_dof_of_action = m.to(self.device)
        self._pd_zero = None
        if len(zero_dofs):
            z = torch.zeros(D, dtype=torch.uint8)
            z[torch.as_tensor(list(zero_dofs), dtype=torch.long)] = 1
            self._pd_zero = z.to(self.device)
        self._pd_tar = torch.zeros(self.num_envs, D, device=self.device)

    def _action_to_pd_targets(self, action: torch.Tensor) -> torch.Tensor:
        """humanoid.py:1711-1713 (+ the reduce_action scatter and the frozen dofs of pre_physics_step, :1540-1556)."""
        if getattr(self, "_pd_action_offset", None) is None:
            raise ops.PhcError("_action_to_pd_targets: call set_pd_action_map(offset, scale, ...) first (the backend owns the dof limits)")
        a = action if (action.dtype == torch.float32 and action.stride(-1) == 1) else action.float().contiguous()
        _lib.check(self._lib.phc_pd_targets(a.data_ptr(), a.stride(0), a.shape[0], self.num_dof, a.shape[1], _ptr(self._pd_dof_of_action),
                                            self._pd_action_offset.data_ptr(), self._pd_action_scale.data_ptr(), _ptr(self._pd_zero),
                                            self._pd_tar.data_ptr(), self._pd_tar.stride(0), _stream()), "phc_pd_targets")
        return self._pd_tar

    def step(self, actions: torch.Tensor) -> None:
        """BaseTask.step (base_task.py:216-234): pre-physics + simulate (backend), then post_physics_step.  With a PD action map
        set the backend receives PD targets (what pre_physics_step hands to gym.set_dof_position_target_tensor), else the raw actions."""
        self.actions = actions
        if actions is not None and getattr(self, "_pd_action_offset", None) is not None:
            actions = self._action_to_pd_targets(actions)
        self.sim.simulate(actions)
        self.post_physics_step()

    @property
    def _amp_obs_buf(self) -> torch.Tensor:
        """Newest-first AMP window [N, S, A] (the reference attribute of that name), materialised from the ring."""
        if self._amp_use_ring:
            ops.amp_window_export(self._amp_store, self._ring_head, self._amp_window)
        return self._amp_window

    def export_amp_obs(self, out: torch.Tensor) -> torch.Tensor:
        """Write extras['amp_obs'] ([N, S*A], newest first) straight into `out` (e.g. the agent's experience-buffer row)."""
        if self._amp_use_ring:
            return ops.amp_window_export(self._amp_store, self._ring_head, out)
        out.copy_(self._amp_store.view(out.shape))
        return out

    def post_physics_step(self) -> None:
        """Humanoid.post_physics_step (humanoid.py:1634-1650) + HumanoidAMP.post_physics_step (humanoid_amp.py:194-210):
        reward, reset, observations, AMP observation -- one launch."""
        self.progress_buf += 1
        if self._amp_use_ring:
            self._plan.advance_ring()
        if self.cycle_motion:
            self._cycle_phase.uniform_()        # what sample_time_interval would draw for the clips that wrap (motion_lib_base.py:415)
        if self._occl_training:
            self._update_occl_training()        # pre_physics_step of the reference (humanoid_im.py:1063-1066)
        if getattr(self, "_eval_mode", False):
            self._plan_eval.run()
            self.extras["terminate"] = self._terminate_buf
            self.extras["reward_raw"] = self.reward_raw
            self.extras["mpjpe"], self.extras["body_pos"], self.extras["body_pos_gt"] = self._plan_eval.mpjpe, self._rigid_body_pos, self._plan_eval.body_pos_gt
            return
        self._plan.run()
        self.extras["terminate"] = self._terminate_buf
        self.extras["reward_raw"] = self.reward_raw
        self.extras["amp_obs_export"] = self.export_amp_obs          # lazily materialised window (see export_amp_obs)
        if self.im_eval:              # kept on the device: the reference's .cpu().numpy() of body_pos / body_pos_gt is the caller's choice
            self.extras["mpjpe"] = self._plan.mpjpe
            self.extras["body_pos"] = self._rigid_body_pos
            self.extras["body_pos_gt"] = self._plan.body_pos_gt

    def _update_occl_training(self) -> None:
        """HumanoidIm._update_occl_training (humanoid_im.py:1081-1092), statement for statement -- including its last two lines, which
        overwrite the sampled pattern with "bodies 0..8 hidden, 9..23 visible" in the reference as shipped."""
        occu = torch.ones(self.num_envs, self.random_occlu_idx.shape[1], device=self.device) * self._occl_training_prob
        idx = torch.bernoulli(occu).bool()
        idx[:, 0] = False
        n = int(idx.shape[0] * idx.shape[1])
        draw = torch.randint(30, 60, (n,), device=self.device).view_as(idx)            # reference: randint of the selected shape (one host sync)
        self.random_occlu_count[:] = torch.where(idx, draw, self.random_occlu_count)
        self.random_occlu_count -= 1
        self.random_occlu_count.clamp_(min=0)
        self.random_occlu_idx[:] = self.random_occlu_count > 0
        self.random_occlu_idx[:] = True
        self.random_occlu_idx[:, 9:24] = False

    # kept for API parity.  Reward, reset and observations of a step are produced TOGETHER by the one fused launch of
    # post_physics_step; these entry points therefore do nothing more (re-launching would advance the AMP ring, decrement
    # _cycle_counter and overwrite _point_goal a second time) and hand back the buffers that launch filled.
    def _compute_reward(self, actions=None):
        return self.rew_buf

    def _compute_reset(self):
        return self.reset_buf

    def _compute_observations(self, env_ids=None):
        self._set_mask(env_ids)
        self._plan_reset_obs.run()
        return self.obs_buf

    def _compute_humanoid_obs(self, env_ids=None):
        """Humanoid._compute_humanoid_obs (humanoid.py:1441-1477): the self observation of the selected envs.  Produced by the
        same observation-only launch as the task observation; returns the `self_obs_buf` rows."""
        self._compute_observations(env_ids)
        return self.self_obs_buf if env_ids is None else self.self_obs_buf[self._reset_mask.bool()]

    def _compute_task_obs(self, env_ids=None, save_buffer=True):
        """HumanoidIm._compute_task_obs (humanoid_im.py:728-871): task observation (v6 or v7) of the selected envs; the ref_body_*
        side buffers are views of the pose cache the launch refreshes (save_buffer is therefore always honoured)."""
        self._compute_observations(env_ids)
        t = self.obs_buf[:, self._plan.self_dim:]
        return t if env_ids is None else t[self._reset_mask.bool()]

    def _compute_amp_observations(self, env_ids=None):
        """HumanoidAMP._compute_amp_observations (humanoid_amp.py:672-707).  The step launch writes the current AMP vector
        itself; outside a step this re-runs it for the current simulator state (all envs, as the reference's env_ids=None)."""
        if env_ids is not None:
            raise NotImplementedError("per-env AMP recomputation outside the fused step: reset paths use phc_amp_obs_demo")
        return self._amp_obs_buf[:, 0]          # slot 0 of the window = the vector the last fused launch wrote

    # ---- reset --------------------------------------------------------------------------------------------------
    def _set_mask(self, env_ids) -> None:
        m = self._reset_mask
        if env_ids is not None and not torch.is_tensor(env_ids):      # the reference also passes lists (done_indices = [], amp_agent.py:314)
            env_ids = torch.as_tensor(env_ids, dtype=torch.int64, device=self.device).reshape(-1)
            m.zero_()
            if env_ids.numel():
                m[env_ids] = 1
            return
        if env_ids is None:
            m.fill_(1)
        elif env_ids.dtype in (torch.bool, torch.uint8, torch.float32) and env_ids.shape == m.shape:
            m.copy_(env_ids != 0)                       # a [N] mask (e.g. dones)
        elif env_ids.dtype == torch.int64 and env_ids.shape == m.shape and m.numel() > 0:
            # [N] int64 is either our own 0/1 mask (reset_buf) or the reference's index list naming every env
            # (`torch.arange(num_envs)`): told apart on the device, without a host sync, by the largest entry
            as_index = torch.zeros_like(m).index_fill_(0, env_ids.clamp(0, m.numel() - 1), 1)
            m.copy_(torch.where(env_ids.max() <= 1, (env_ids != 0).to(m.dtype), as_index))
        else:                                           # reference-style index list
            m.zero_()
            m[env_ids] = 1

    def _sample_time(self, motion_ids: torch.Tensor) -> torch.Tensor:
        """MotionLibBase.sample_time_interval (motion_lib_base.py:414-423): start times on the 1/30 s grid."""
        phase = torch.rand(motion_ids.shape, device=self.device)
        ln = self._motion_lib.lengths[motion_ids]
        return ((phase * ln) / (1.0 / 30.0)).long() * (1.0 / 30.0)

    def reset(self, env_ids=None) -> torch.Tensor:
        """Humanoid.reset -> _reset_envs (humanoid.py:537-621, humanoid_amp.py:378-387,:509-603, humanoid_im.py:955-1023)
        with reference-state initialisation, for the envs selected by `env_ids` (None = all, a [N] mask, or indices)."""
        self._set_mask(env_ids)
        lib, ml, st = self._lib, self._motion_lib, _stream()
        # new start time (sample_time_interval) + cleared counters of the selected envs: one launch
        phase = torch.rand(self.num_envs, device=self.device)
        if getattr(self, "_eval_mode", False) or bool(self.cfg.get("test", False)):
            phase.zero_()                                 # flags.test: motion_times[:] = 0 (humanoid_im.py:1010-1011)
        _lib.check(lib.phc_reset_bookkeeping(self._reset_mask.data_ptr(), phase.data_ptr(), self._plan._env_motion.data_ptr(), self.num_envs,
                                             self._motion_start_times.data_ptr(), self._motion_start_times_offset.data_ptr(),
                                             self._global_offset.data_ptr(), self._cycle_counter.data_ptr(), self.progress_buf.data_ptr(),
                                             self.reset_buf.data_ptr(), self._terminate_buf.data_ptr(), st), "phc_reset_bookkeeping")
        # _set_env_state: reference pose at the sampled time into the simulator tensors of the reset envs
        _lib.check(lib.phc_set_env_state(C.byref(ml.c), self._sampled_motion_ids.data_ptr(), self._motion_start_times.data_ptr(),
                                         self._global_offset.data_ptr(), self._reset_mask.data_ptr(), self.num_envs,
                                         self._rigid_body_state_reshaped.data_ptr(), self.sim.bodies_per_env,
                                         self._dof_state.data_ptr(), st), "phc_set_env_state")
        # _reset_env_tensors (humanoid.py:590-621): the backend pushes the new root / dof state of the flagged envs into the simulation
        # (Isaac Gym: set_actor_root_state_tensor_indexed + set_dof_state_tensor_indexed on mask.nonzero() in ITS reset path)
        self.sim.set_env_state(self._reset_mask, self._rigid_body_state_reshaped, self._dof_state)
        # _compute_observations(env_ids)
        self._plan_reset_obs.run()
        # _init_amp_obs: current + history slots from the reference motion at t0 - k dt
        ops.amp_obs_demo(ml, self.step_cfg, self._sampled_motion_ids, self._motion_start_times, first_step=0,
                         num_steps=self._num_amp_obs_steps, out=self._amp_store, only_where=self._reset_mask,
                         slot_offset=0, slot_offset_dev=self._ring_head)
        return self.obs_buf

    def _load_motion(self, env, sim):
        """Humanoid._load_motion for humanoid_type smpl (humanoid_im.py:300-341): MotionLibSMPL over env.motion_file, one clip per env
        loaded with the per-env skeleton trees / shapes / limb weights the simulator side built from its assets."""
        from ..motion_lib import MotionLibSMPL
        motion_file = env.get("motion_file", self.cfg.get("motion_file", None))
        if motion_file is None:
            raise KeyError("HumanoidIm: cfg has neither `motion_data` (pre-built tables) nor env.motion_file")
        for need in ("skeleton_trees", "humanoid_shapes", "humanoid_limb_and_weights"):
            if not hasattr(sim, need):
                raise TypeError(f"HumanoidIm: loading {motion_file!r} needs the backend's `{need}` (Humanoid keeps them per env, humanoid.py:780-860)")
        self.seq_motions = bool(env.get("seq_motions", False))
        self.max_len = int(env.get("max_len", -1)) if "max_len" in env else -1
        self._min_motion_len = int(env.get("min_length", -1))
        test = bool(self.cfg.get("test", False))
        lib = MotionLibSMPL(dict(motion_file=motion_file, device=self.device, fix_height=0, min_length=self._min_motion_len, max_length=self.max_len,
                                 im_eval=bool(self.cfg.get("im_eval", False)), multi_thread=False, smpl_type=self._rcfg("humanoid_type", "smpl"),
                                 randomrize_heading=True, step_dt=self.dt, test=test))
        self._motion_train_lib = self._motion_eval_lib = lib
        lib.load_motions(skeleton_trees=sim.skeleton_trees, gender_betas=torch.as_tensor(sim.humanoid_shapes).cpu(),
                         limb_weights=torch.as_tensor(sim.humanoid_limb_and_weights).cpu(), random_sample=(not test) and (not self.seq_motions),
                         max_len=-1 if test else self.max_len)
        return lib

    def _reload_motions(self, random_sample: bool, start_idx: int = 0) -> None:
        """MotionLib.load_motions with the simulator side's per-env assets, then both launch plans re-pointed at the new tables."""
        lib = self._motion_data
        test = bool(self.cfg.get("test", False))
        lib.load_motions(skeleton_trees=self.sim.skeleton_trees, gender_betas=torch.as_tensor(self.sim.humanoid_shapes).cpu(),
                         limb_weights=torch.as_tensor(self.sim.humanoid_limb_and_weights).cpu(), random_sample=random_sample, start_idx=start_idx,
                         max_len=-1 if (test or not random_sample) else getattr(self, "max_len", -1))
        self._motion_lib = lib.packed
        self._motion_version = getattr(self, "_motion_version", 0) + 1      # a graph-captured rollout of the agent has to be re-captured
        for plan in (self._plan, self._plan_reset_obs, getattr(self, "_plan_eval", None)):
            if plan is not None:
                plan.set_motion_lib(self._motion_lib)

    def resample_motions(self):
        """HumanoidIm.resample_motions (humanoid_im.py:369-394).  With a loadable library (`MotionLibSMPL.load_motions`): sample and load a
        new set of clips on the device, re-point the launch plans at the new tables, keep every humanoid where it stands
        (`_global_offset[:, :2] = root xy - reference root xy at the env's current motion time`), reset all envs.  With fixed tables
        (synthetic data) only the per-env motion records are refreshed (`_sampled_motion_ids` may have been edited)."""
        lib = self._motion_data
        if hasattr(lib, "load_motions") and hasattr(self.sim, "skeleton_trees"):
            test = bool(self.cfg.get("test", False))
            self._reload_motions(random_sample=(not test) and (not getattr(self, "seq_motions", False)))
            t = self.progress_buf.float() * self.dt + self._motion_start_times + self._motion_start_times_offset
            root = ops.motion_state(self._motion_lib, self._sampled_motion_ids, t.contiguous(), want_dof=False)["root_pos"]   # get_root_pos_smpl
            self._global_offset[:, :2] = self._rigid_body_state_reshaped[:, 0, :2] - root[:, :2]
            self.reset()
            return
        self._plan.refresh_motion_params()
        self._plan_reset_obs.refresh_motion_params()

    # ---- evaluation (IMAmpAgent.eval, im_amp.py:136-242) ----------------------------------------------------------
    def begin_seq_motion_samples(self):
        """humanoid_im.py:468-472: clips in dataset order from the start (not sampled), all envs reset at motion time 0."""
        self.start_idx = 0
        self._reload_motions(random_sample=False, start_idx=0)
        self.reset()

    def forward_motion_samples(self):
        """humanoid_im.py:474-477: the next num_envs clips of the dataset."""
        self.start_idx += self.num_envs
        self._reload_motions(random_sample=False, start_idx=self.start_idx)
        self.reset()

    def set_eval_mode(self, on: bool, termination_distance: float = 0.5) -> None:
        """What IMAmpAgent.eval switches on the task and back (im_amp.py:160-184, :226-238): every termination distance 0.5 (UHC's),
        mean-distance termination unless strict_eval (`flags.im_eval`, humanoid_im.py:1180), the mpjpe / body_pos_gt extras, no clip
        cycling, no far-reference handling, resets at motion time 0 (`flags.test`, :1010-1011).  Implemented as a second launch plan over
        the SAME buffers, built once; `step()` uses it while the mode is on."""
        self._eval_mode = bool(on)
        if on and getattr(self, "_plan_eval", None) is None:
            import dataclasses
            env = self.cfg.get("env", self.cfg)
            J = self.num_bodies
            rb = list(self._reset_bodies_id) if self._reset_bodies_id is not None else list(range(J))
            if len(rb) > 15 and env.get("eval_body_ids") is not None:        # "Following UHC": the eval subset for full-body tracking (:182-183)
                rb = [int(b) for b in env["eval_body_ids"]]
            cfg_eval = dataclasses.replace(self.step_cfg, term_dist=float(termination_distance), reset_bodies=rb, cycle_motion=False, zero_out_far=False,
                                           term_use_mean=not bool(env.get("strict_eval", False)), specialise=False)
            p = self._plan
            self._plan_eval = ops.EnvStepPlan(cfg_eval, self._motion_lib, self._rigid_body_state_reshaped, self._dof_state, self.dof_force_tensor,
                                              self.progress_buf, self._sampled_motion_ids, self._motion_start_times, self._motion_start_times_offset,
                                              self._global_offset, cycle_counter=self._cycle_counter, obs=self.obs_buf, rew=self.rew_buf,
                                              reward_raw=self.reward_raw, reset=self.reset_buf, terminate=self._terminate_buf,
                                              amp_obs_buf=self._amp_store, amp_ring=self._amp_use_ring, ring_head_dev=self._ring_head,
                                              ref_cache=self._ref_cache, reward_from_cache=self._use_ref_cache, with_eval_extras=True,
                                              occlusion=self.random_occlu_idx, shape_params=p._keep.get("shape_params"),
                                              limb_weights=p._keep.get("limb_weights"))

    # ---- discriminator demo observations ------------------------------------------------------------------------
    def fetch_amp_obs_demo(self, num_samples: int) -> torch.Tensor:
        """HumanoidAMP.fetch_amp_obs_demo (humanoid_amp.py:215-230): AMP windows of random reference-motion states."""
        sample = getattr(self._motion_data, "sample_motions", None)
        if sample is not None:         # MotionLibBase.sample_motions: multinomial over _sampling_batch_prob (Auto-PMCP re-weights it)
            ids = sample(num_samples).to(self.device, torch.int64)
        else:                          # plain tables (synthetic data): every clip equally likely, as an un-weighted library
            ids = torch.randint(0, self._motion_lib.num_motions, (num_samples,), device=self.device)
        t0 = self._sample_time(ids).float()          # HumanoidIm._sample_time -> sample_time_interval (humanoid_im.py:661-663)
        demo = ops.amp_obs_demo(self._motion_lib, self.step_cfg, ids, t0)
        return demo.view(num_samples, self.get_num_amp_obs())


class VecTaskPythonWrapper:
    """phc/env/tasks/vec_task_wrappers.py:45-81 + VecTaskPython (vec_task.py:150-166)."""

    def __init__(self, task: HumanoidIm, clip_observations: float = float("inf")):
        self.task = task
        self.clip_obs = clip_observations
        self.num_envs = task.num_envs

    def step(self, actions):
        self.task.step(actions)
        obs = self.task.obs_buf
        if self.clip_obs != float("inf"):
            obs = torch.clamp(obs, -self.clip_obs, self.clip_obs)
        return obs, self.task.rew_buf, self.task.reset_buf, self.task.extras

    def reset(self, env_ids=None):
        return self.task.reset(env_ids)

    def fetch_amp_obs_demo(self, num_samples):
        return self.task.fetch_amp_obs_demo(num_samples)


class RLGPUEnv:
    """phc/run_hydra.py:187-240: the vec-env object the agent holds (`vec_env.env.task` is the HumanoidIm)."""

    def __init__(self, task: HumanoidIm):
        self.env = VecTaskPythonWrapper(task)

    def step(self, action):
        obs, rew, reset, extras = self.env.step(action)
        return {"obs": obs}, rew, reset, extras      # extras['amp_obs_export'](dst) fills the AMP window (amp_agent.py:341)

    def reset(self, env_ids=None):
        return {"obs": self.env.reset(env_ids)}

    def get_env_info(self):
        t = self.env.task
        return dict(num_obs=t.get_obs_size(), num_actions=t.get_action_size(), num_amp_obs=t.get_num_amp_obs())
