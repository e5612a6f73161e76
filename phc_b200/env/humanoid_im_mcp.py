"""HumanoidImMCP: the multiplicative-composer task (phc/env/tasks/humanoid_im_mcp.py).

The agent's action is a weight vector over `num_prim` frozen primitives; the env normalises its own observation with the
primitives' running statistics, evaluates every primitive, mixes their PD targets with the weights and then steps as
HumanoidIm does.  Device work per step: phc_rms_apply -> K x 3 tensor-core GEMMs -> phc_mcp_combine -> fused env step.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from .. import _lib
from ..learning.amp_agent import RunningMeanStd, _stream
from ..learning.network_loader import FrozenPNN, load_pnn
from .humanoid_im import HumanoidIm


class HumanoidImMCP(HumanoidIm):

    def __init__(self, cfg: Dict, sim_params=None, physics_engine=None, device_type: str = "cuda", device_id: int = 0,
                 headless: bool = True, pnn_checkpoint: Optional[Dict] = None):
        env = cfg.get("env", cfg)
        self.num_prim = env.get("num_prim", 3)
        self.discrete_mcp = env.get("discrete_moe", False)
        self.has_pnn = env.get("has_pnn", False)
        self.has_lateral = env.get("has_lateral", False)
        self.z_activation = env.get("z_activation", "relu")
        super().__init__(cfg, sim_params, physics_engine, device_type, device_id, headless)
        if not self.has_pnn:
            raise NotImplementedError("has_pnn: False (separately loaded actors) is not used by the shipped MCP configs")
        if pnn_checkpoint is None:                                  # humanoid_im_mcp.py:26-29
            paths = env.get("models", [])
            assert len(paths) == 1
            pnn_checkpoint = torch.load(paths[0], map_location="cpu")
        self.pnn: FrozenPNN = load_pnn(pnn_checkpoint, num_prim=self.num_prim, has_lateral=self.has_lateral,
                                       activation=self.z_activation, device=self.device)
        rms = pnn_checkpoint["running_mean_std"]
        self._pnn_rms = RunningMeanStd(self.get_obs_size(), self.device, epsilon=1e-5)
        self._pnn_rms.running_mean.copy_(rms["running_mean"].to(self.device, torch.float64))
        self._pnn_rms.running_var.copy_(rms["running_var"].to(self.device, torch.float64))
        self._pnn_rms.freeze()
        self.running_mean, self.running_var = rms["running_mean"], rms["running_var"]
        self._mixed = torch.zeros(self.num_envs, self.num_dof, dtype=torch.float32, device=self.device)
        self._lib = _lib.load()

    def get_action_size(self):
        return self.num_prim                                        # _setup_character_props (humanoid_im_mcp.py:45-48)

    def get_task_obs_size_detail(self):
        d = super().get_task_obs_size_detail()
        d["num_prim"] = self.num_prim
        return d

    def compose_actions(self, weights: torch.Tensor) -> torch.Tensor:
        """humanoid_im_mcp.py:64-82: clamp((obs - mean)/sqrt(var + 1e-5), +-5) -> all primitives -> sum_k w_k a_k."""
        N = self.num_envs
        x = self.pnn.input_buffer(N)
        self._pnn_rms.apply(self.obs_buf, x)
        prim = self.pnn.forward_all(x)                              # [K, N, ld]
        w = weights if weights.dtype == torch.float32 and weights.stride(-1) == 1 else weights.float().contiguous()
        rc = self._lib.phc_mcp_combine(w.data_ptr(), w.stride(0), prim.data_ptr(), prim.stride(1), prim.stride(0), N, self.num_prim,
                                       self.num_dof, 1 if self.discrete_mcp else 0, self._mixed.data_ptr(), self._mixed.stride(0),
                                       _stream())
        if rc:
            _lib.check(rc, "phc_mcp_combine")
        return self._mixed

    def step(self, weights: torch.Tensor) -> None:
        actions = self.compose_actions(weights)
        self.actions = actions
        if getattr(self, "_pd_action_offset", None) is not None:        # mixed action -> PD targets (humanoid.py:1711-1713)
            actions = self._action_to_pd_targets(actions)
        self.sim.simulate(actions)
        self.post_physics_step()
