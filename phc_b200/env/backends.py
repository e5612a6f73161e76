"""Simulator backends of HumanoidIm.

The rigid-body simulator is not part of phc_b200: `HumanoidIm` reads the tensors a backend exposes and asks it to advance the
physics.  What a backend is (duck typed; `SyntheticSim` in humanoid_im.py and `IsaacGymBackend` below are the two in the tree):

    rigid_body_state  [N, bodies_per_env, 13] fp32   pos3 rot4(xyzw) vel3 angvel3        (Humanoid._setup_tensors, humanoid.py:219-226)
    dof_state         [N, D, 2] fp32                 (pos, vel)                          (humanoid.py:211-214)
    dof_force         [N, D] fp32                                                        (humanoid.py:193-194)
    bodies_per_env    int
    simulate(actions)                      pre_physics_step + gym.simulate + refresh of the tensors above (base_task.py:216-231)
    set_env_state(mask, rigid_body_state, dof_state)
                                           push the rows HumanoidIm.reset rewrote into the simulation (humanoid.py:590-621)
  optional, needed when HumanoidIm has to LOAD motions itself (cfg without `motion_data`):
    skeleton_trees, humanoid_shapes, humanoid_limb_and_weights       what Humanoid keeps per env for MotionLib.load_motions
  optional:
    generate_fall_states()                 -> (root_states [N, 13], dof_pos [N, D]): the bank of fallen states HumanoidImGetup starts
                                           episodes from (humanoid_im_getup.py:82-125); required by HumanoidImGetup / HumanoidImMCPGetup
    pd_action_offset / pd_action_scale     Humanoid._build_pd_action_offset_scale (humanoid.py:1331-1380)
    graph_safe = True                      simulate() only enqueues work on the current CUDA stream (CUDA-graph capturable)

When the reference's own entry point constructs the task (`eval(args.task)(cfg=cfg, sim_params=..., physics_engine=..., ...)`,
parse_task.py:60) nobody hands a backend over, so a FACTORY does: phc_b200.dropin registers one that instantiates the reference's
original task class (saved before the rebinding) as the owner of gym / sim / assets and wraps it in `IsaacGymBackend`.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

_FACTORY: Optional[Callable] = None


def register_backend_factory(fn: Optional[Callable]) -> None:
    """fn(cfg, sim_params, physics_engine, device_type, device_id, headless) -> backend.  None clears it."""
    global _FACTORY
    _FACTORY = fn


def make_backend(cfg, sim_params, physics_engine, device_type, device_id, headless):
    if _FACTORY is None:
        raise RuntimeError(
            "HumanoidIm: no simulator backend.  Pass one as cfg['sim_backend'] (an object with rigid_body_state / dof_state / dof_force / "
            "simulate / set_env_state, see phc_b200/env/backends.py), pass synthetic `motion_data` to get the SyntheticSim stand-in, or "
            "register a factory (phc_b200.env.backends.register_backend_factory; phc_b200.dropin.install() registers the Isaac Gym one "
            "when the reference task module is importable).  There is no silent fallback.")
    return _FACTORY(cfg, sim_params, physics_engine, device_type, device_id, headless)


class IsaacGymBackend:
    """The reference's own task instance as the physics owner (gym, sim, assets, actors): everything HumanoidIm replaces -- observations,
    reward, reset logic, motion library -- is simply not called on it; `simulate` is BaseTask.step minus post_physics_step."""

    graph_safe = False          # gym.simulate is not a CUDA-stream operation

    def __init__(self, ref_task):
        t = self._t = ref_task
        self.rigid_body_state = t._rigid_body_state_reshaped
        self.dof_state = t._dof_state.view(t.num_envs, -1, 2)
        self.dof_force = t.dof_force_tensor
        self.bodies_per_env = int(self.rigid_body_state.shape[1])
        for name in ("skeleton_trees", "humanoid_shapes", "humanoid_limb_and_weights"):
            if hasattr(t, name):
                setattr(self, name, getattr(t, name))
        if hasattr(t, "_pd_action_offset"):
            self.pd_action_offset, self.pd_action_scale = t._pd_action_offset, t._pd_action_scale

    def simulate(self, actions) -> None:
        t = self._t
        t.pre_physics_step(actions)
        t._physics_step()
        t._refresh_sim_tensors()

    def set_env_state(self, mask: torch.Tensor, rigid_body_state: torch.Tensor, dof_state: torch.Tensor) -> None:
        """Humanoid._reset_env_tensors (humanoid.py:590-621): root + dof state of the flagged envs into the simulation."""
        from isaacgym import gymtorch
        t = self._t
        ids = mask.nonzero(as_tuple=False).flatten()
        if ids.numel() == 0:
            return
        t._humanoid_root_states[ids] = rigid_body_state[ids, 0]
        actor_ids = t._humanoid_actor_ids[ids]
        t.gym.set_actor_root_state_tensor_indexed(t.sim, gymtorch.unwrap_tensor(t._root_states), gymtorch.unwrap_tensor(actor_ids), len(actor_ids))
        t.gym.set_dof_state_tensor_indexed(t.sim, gymtorch.unwrap_tensor(t._dof_state), gymtorch.unwrap_tensor(actor_ids), len(actor_ids))

    def generate_fall_states(self):
        """HumanoidImGetup._generate_fall_states (humanoid_im_getup.py:82-125) on the wrapped task: random unit root rotations at the
        initial root states, zero dof state, one uniform [-0.5, 0.5) action, 150 physics steps; returns the settled root states (velocities
        zeroed) and dof positions."""
        import numpy as np
        from isaacgym import gymtorch
        t = self._t
        N = t.num_envs
        env_ids = torch.arange(N, device=t.device, dtype=torch.long)
        root_states = t._initial_humanoid_root_states[env_ids].clone()
        root_states[..., 3:7] = torch.randn_like(root_states[..., 3:7])
        root_states[..., 3:7] = torch.nn.functional.normalize(root_states[..., 3:7], dim=-1)
        t._humanoid_root_states[env_ids] = root_states
        actor_ids = t._humanoid_actor_ids[env_ids]
        t.gym.set_actor_root_state_tensor_indexed(t.sim, gymtorch.unwrap_tensor(t._root_states), gymtorch.unwrap_tensor(actor_ids), len(actor_ids))
        t.gym.set_dof_state_tensor_indexed(t.sim, gymtorch.unwrap_tensor(torch.zeros_like(t._dof_state)), gymtorch.unwrap_tensor(actor_ids),
                                           len(actor_ids))
        rand_actions = torch.as_tensor(np.random.uniform(-0.5, 0.5, size=[N, t.get_dof_action_size()]), dtype=torch.float32, device=t.device)
        t.pre_physics_step(rand_actions)
        for _ in range(150):
            t.render()
            t.gym.simulate(t.sim)
        t._refresh_sim_tensors()
        root = t._humanoid_root_states.clone()
        root[:, 7:13] = 0
        return root, t._dof_pos.clone()
