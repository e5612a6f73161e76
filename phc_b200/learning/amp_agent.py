"""AMPAgent: PPO + AMP discriminator training loop on the phc_b200 kernels.

Mirrors the API surface of the reference agent stack so it can stand in for it behind rl_games' runner:
  CommonAgent (phc/learning/common_agent.py): train / train_epoch / play_steps / discount_values / _calc_advs /
      prepare_dataset / get_action_values / _eval_critic / bound_loss / _actor_loss / _critic_loss
  AMPAgent    (phc/learning/amp_agent.py): calc_gradients / _disc_loss / _calc_amp_rewards / _combine_rewards /
      _preproc_obs / _preproc_amp_obs / get_stats_weights / set_stats_weights / get_full_state_weights / ...
rl_games==1.1.4 (the real base class, not in the reference tree) is restated where the hot path needs it:
ExperienceBuffer (time-major [T, N, ...]), swap_and_flatten01, Adam + clip_grad_norm_, Horovod grad averaging
(-> one NCCL all-reduce on the flat gradient bucket per minibatch).

What runs where: every tensor op on the path is a libphc_b200.so kernel (GEMMs, normalisers, losses, GAE, Adam);
torch supplies memory, RNG (randn / randperm) and torch.distributed.
"""
from __future__ import annotations

import copy
import os
import time
from typing import Dict, Optional

import torch

from .. import _lib, ops
from ..ops import _ptr, _stream
from . import dist as D
from .networks import AMPNetwork, MLPEngine, round4

DEFAULT_CONFIG = dict(          # phc/data/cfg/learning/im.yaml:43-99
    name="Humanoid", multi_gpu=False, normalize_input=True, normalize_value=True, normalize_advantage=True,
    gamma=0.99, tau=0.95, learning_rate=2e-5, truncate_grads=True, grad_norm=50.0, e_clip=0.2, horizon_length=32,
    minibatch_size=16384, mini_epochs=6, critic_coef=5.0, clip_value=False, bounds_loss_coef=10.0, entropy_coef=0.0,
    amp_obs_demo_buffer_size=200000, amp_replay_buffer_size=200000, amp_replay_keep_prob=0.01, amp_batch_size=512,
    amp_minibatch_size=4096, disc_coef=5.0, disc_logit_reg=0.01, disc_grad_penalty=5.0, disc_reward_scale=2.0,
    disc_weight_decay=0.0001, normalize_amp_input=True, task_reward_w=0.5, disc_reward_w=0.5, max_epochs=10000000,
    save_frequency=2500, save_best_after=100, seed=0,
    network=dict(mlp=dict(units=[1024, 512], activation="relu"), disc=dict(units=[1024, 512], activation="relu"),
                 sigma_init=-2.9),
)


class PhaseTimer:
    """Optional CUDA-event phase breakdown of an epoch (PHC_PHASE_TIMING=1): `with timer("name"):` records an event pair on
    the current stream; `report()` synchronises once and returns {name: milliseconds}.  Disabled = zero overhead."""

    class _Span:
        def __init__(self, owner, name):
            self.o, self.n = owner, name

        def __enter__(self):
            if self.o.enabled:
                self.e0 = torch.cuda.Event(enable_timing=True)
                self.e0.record()

        def __exit__(self, *a):
            if self.o.enabled:
                e1 = torch.cuda.Event(enable_timing=True)
                e1.record()
                self.o.spans.append((self.n, self.e0, e1))

    def __init__(self, enabled: bool):
        self.enabled = enabled
        self.spans = []

    def __call__(self, name):
        return PhaseTimer._Span(self, name)

    def report(self):
        torch.cuda.synchronize()
        out = {}
        for n, a, b in self.spans:
            out[n] = out.get(n, 0.0) + a.elapsed_time(b)
        self.spans = []
        return out


class RunningMeanStd:
    """phc/utils/running_mean_std.py: fp64 running mean / var / count on the device, kernels phc_rms_apply/update."""

    def __init__(self, size: int, device, epsilon: float = 1e-5):
        self.size, self.epsilon, self.device = int(size), epsilon, torch.device(device)
        self.running_mean = torch.zeros(size, dtype=torch.float64, device=self.device)
        self.running_var = torch.ones(size, dtype=torch.float64, device=self.device)
        self.count = torch.ones((), dtype=torch.float64, device=self.device)
        self.frozen = False
        self.training = True
        self._lib = _lib.load()
        self._ws = torch.zeros(self._lib.phc_rms_workspace_bytes(self.size) // 8, dtype=torch.float64, device=self.device)

    def train(self):
        self.training = True

    def eval(self):
        self.training = False

    def freeze(self):
        self.frozen = True

    def frozen_copy(self) -> "RunningMeanStd":
        c = RunningMeanStd(self.size, self.device, self.epsilon)
        c.running_mean.copy_(self.running_mean)
        c.running_var.copy_(self.running_var)
        c.count.copy_(self.count)
        c.frozen = True
        return c

    def apply(self, x: torch.Tensor, out: torch.Tensor, unnorm: bool = False, row_idx: Optional[torch.Tensor] = None,
              n: Optional[int] = None) -> torch.Tensor:
        n = (x.shape[0] if row_idx is None else row_idx.shape[0]) if n is None else n
        rc = self._lib.phc_rms_apply(x.data_ptr(), x.stride(0), n, self.size, self.running_mean.data_ptr(),
                                     self.running_var.data_ptr(), self.epsilon, 1 if unnorm else 0, out.data_ptr(),
                                     out.stride(0), _ptr(row_idx), _stream())
        if rc:
            _lib.check(rc, "phc_rms_apply")
        return out

    def apply_update(self, x: torch.Tensor, out: torch.Tensor, row_idx: Optional[torch.Tensor] = None, n: Optional[int] = None,
                     apply_stats: Optional["RunningMeanStd"] = None) -> torch.Tensor:
        """apply() with `apply_stats` (default: these statistics, as they are BEFORE the update) and update() of these statistics in one
        pass over the rows (phc_rms_apply_update): RunningMeanStd.forward in train mode / _preproc_obs(use_temp=True)."""
        n = (x.shape[0] if row_idx is None else row_idx.shape[0]) if n is None else n
        a = self if apply_stats is None else apply_stats
        rc = self._lib.phc_rms_apply_update(x.data_ptr(), x.stride(0), n, self.size, a.running_mean.data_ptr(), a.running_var.data_ptr(), a.epsilon,
                                            out.data_ptr(), out.stride(0), _ptr(row_idx), self.running_mean.data_ptr(), self.running_var.data_ptr(),
                                            self.count.data_ptr(), self._ws.data_ptr(), _stream())
        if rc:
            _lib.check(rc, "phc_rms_apply_update")
        return out

    def update(self, x: torch.Tensor, n: Optional[int] = None, row_idx: Optional[torch.Tensor] = None) -> None:
        n = (x.shape[0] if row_idx is None else row_idx.shape[0]) if n is None else n
        rc = self._lib.phc_rms_update(x.data_ptr(), x.stride(0), n, self.size, self.running_mean.data_ptr(),
                                      self.running_var.data_ptr(), self.count.data_ptr(), self._ws.data_ptr(),
                                      _ptr(row_idx), _stream())
        if rc:
            _lib.check(rc, "phc_rms_update")

    def __call__(self, x: torch.Tensor, unnorm: bool = False) -> torch.Tensor:
        """RunningMeanStd.forward: normalise (then, in train mode and not frozen, fold the batch into the stats)."""
        x2 = x.reshape(-1, self.size)
        out = torch.empty_like(x2)
        self.apply(x2, out, unnorm)
        if self.training and not self.frozen and not unnorm:
            self.update(x2)
        return out.view(x.shape)

    def state_dict(self):
        return {"running_mean": self.running_mean.clone(), "running_var": self.running_var.clone(), "count": self.count.clone()}

    def load_state_dict(self, sd):
        self.running_mean.copy_(sd["running_mean"].to(self.device))
        self.running_var.copy_(sd["running_var"].to(self.device))
        self.count.copy_(sd["count"].to(self.device))


class ReplayBuffer:
    """phc/learning/replay_buffer.py with index-returning sampling (rows are gathered later, once, by the consumer)."""

    def __init__(self, buffer_size: int, width: int, device):
        self._size, self._head, self._total, self.device = int(buffer_size), 0, 0, torch.device(device)
        self.data = torch.zeros(self._size, width, dtype=torch.float32, device=self.device)
        self._sample_idx = torch.randperm(self._size, device=self.device)
        self._sample_head = 0

    def get_buffer_size(self):
        return self._size

    def get_total_count(self):
        return self._total

    def store(self, rows: torch.Tensor) -> None:
        n = rows.shape[0]
        assert n <= self._size
        first = min(n, self._size - self._head)
        self.data[self._head:self._head + first] = rows[:first]
        if n > first:
            self.data[0:n - first] = rows[first:]
        self._head = (self._head + n) % self._size
        self._total += n

    def sample_indices(self, n: int) -> torch.Tensor:
        idx = (torch.arange(self._sample_head, self._sample_head + n, device=self.device)) % self._size
        rand_idx = self._sample_idx[idx]
        if self._total < self._size:
            rand_idx = rand_idx % self._head
        self._sample_head += n
        if self._sample_head >= self._size:
            self._sample_idx = torch.randperm(self._size, device=self.device)
            self._sample_head = 0
        return rand_idx


def task_detail(task, key: str, default: int) -> int:
    """AMPPNNBuilder / AMPMCPBuilder read num_prim / training_prim from the task's obs-size detail
    (amp_network_pnn_builder.py:33-36, amp_network_mcp_builder.py:40)."""
    fn = getattr(task, "get_task_obs_size_detail", None)
    return int(fn().get(key, default)) if fn is not None else default


class AMPAgent:
    def __init__(self, base_name: str, config: Dict):
        cfg = copy.deepcopy(DEFAULT_CONFIG)
        cfg.update({k: v for k, v in config.items() if k != "network"})
        if "network" in config:
            cfg["network"].update(self._network_spec(config["network"]))     # a dict, or rl_games' model / builder object
        self.config = cfg
        self.base_name = base_name
        self.vec_env = cfg.get("vec_env") or self._create_vec_env(cfg)
        task = self.vec_env.env.task
        self.device = torch.device(cfg.get("device", task.device))
        self.ppo_device = self.device
        torch.cuda.set_device(self.device)
        self._lib = _lib.load()

        self.num_actors = task.num_envs
        self.num_agents = 1
        self.horizon_length = int(cfg["horizon_length"])
        self.batch_size = self.horizon_length * self.num_actors
        self.minibatch_size = min(int(cfg["minibatch_size"]), self.batch_size)
        assert self.batch_size % self.minibatch_size == 0
        self.num_minibatches = self.batch_size // self.minibatch_size
        self.mini_epochs_num = int(cfg["mini_epochs"])
        self.gamma, self.tau, self.e_clip = float(cfg["gamma"]), float(cfg["tau"]), float(cfg["e_clip"])
        self.last_lr = float(cfg["learning_rate"])
        self.critic_coef, self.bounds_loss_coef = float(cfg["critic_coef"]), float(cfg["bounds_loss_coef"])
        self.entropy_coef = float(cfg["entropy_coef"])
        self.truncate_grads, self.grad_norm = bool(cfg["truncate_grads"]), float(cfg["grad_norm"])
        self.normalize_input, self.normalize_value = bool(cfg["normalize_input"]), bool(cfg["normalize_value"])
        self.normalize_advantage = bool(cfg["normalize_advantage"])
        self._task_reward_w, self._disc_reward_w = float(cfg["task_reward_w"]), float(cfg["disc_reward_w"])
        self._amp_batch_size = int(cfg["amp_batch_size"])
        self._amp_minibatch_size = min(int(cfg["amp_minibatch_size"]), self.minibatch_size)
        self._disc_coef, self._disc_logit_reg = float(cfg["disc_coef"]), float(cfg["disc_logit_reg"])
        self._disc_grad_penalty, self._disc_weight_decay = float(cfg["disc_grad_penalty"]), float(cfg["disc_weight_decay"])
        self._disc_reward_scale = float(cfg["disc_reward_scale"])
        self._normalize_amp_input = bool(cfg["normalize_amp_input"])
        self._amp_replay_keep_prob = float(cfg["amp_replay_keep_prob"])
        self.temp_running_mean = getattr(task, "temp_running_mean", True)

        self.obs_dim = task.get_obs_size()
        self.actions_num = task.get_action_size()
        self.amp_obs_dim = task.get_num_amp_obs()
        self.obs_pad, self.amp_pad, self.act_pad = round4(self.obs_dim), round4(self.amp_obs_dim), round4(self.actions_num)

        # multi-GPU: one process per GPU, gradients summed over NCCL and scaled by 1/world (replaces Horovod,
        # phc/run_hydra.py:114-128 / amp_agent.py:668)
        self.multi_gpu = bool(cfg.get("multi_gpu", False)) and D.is_multi()
        self._reducer = D.GradReducer(self.device)
        self.rank = torch.distributed.get_rank() if self.multi_gpu else 0
        self.world = D.world_size() if self.multi_gpu else 1

        netcfg = cfg["network"] = self._network_spec(cfg["network"])
        if netcfg.get("name", "amp") == "amp_mcp":
            # AMPMCPBuilder (amp_network_mcp_builder.py:33-59): has_softmax defaults to TRUE there (appends nn.Softmax) and
            # ending_act False strips the final activation.  The shipped MCP configs set has_softmax: False with ending_act: True
            # (im_mcp.yaml:15-16, im_mcp_big.yaml:15-16); phc_comp_kp_2 runs im_mcp_big with ending_act: False (a linear head).
            # The softmax composer must not be built silently.
            if bool(netcfg.get("has_softmax", True)):
                raise NotImplementedError("amp_mcp composer: only has_softmax: False (im_mcp.yaml / im_mcp_big.yaml) is implemented; "
                                          "set it explicitly in the network config")
        self.model = AMPNetwork(self.obs_dim, self.actions_num, self.amp_obs_dim, netcfg["mlp"]["units"],
                                netcfg["disc"]["units"], netcfg["mlp"]["activation"], netcfg.get("sigma_init", -2.9),
                                device=self.device, seed=int(cfg["seed"]),
                                # network.name of the yaml: amp (im.yaml), amp_pnn (im_pnn.yaml), amp_mcp (im_mcp.yaml)
                                kind=netcfg.get("name", "amp"), num_prim=int(netcfg.get("num_prim", task_detail(task, "num_prim", 4))),
                                training_prim=int(netcfg.get("training_prim", task_detail(task, "training_prim", 0))),
                                ending_act=bool(netcfg.get("ending_act", True)))
        if self.multi_gpu:
            D.broadcast_params(self.model.params, 0)
            self.model.refresh_images()                 # the collective wrote the bucket behind torch's version counter
        # mlp_precision: "fp32" (3xTF32, the reference's mixed_precision: False) or "tf32" (single tensor-core pass, opt-in)
        self.engine = MLPEngine(self.model, precision=str(cfg.get("mlp_precision", "fp32")))
        n = self.model.num_floats
        self.exp_avg = torch.zeros(n, device=self.device)
        self.exp_avg_sq = torch.zeros(n, device=self.device)
        self.opt_step = 0
        self._gsumsq = torch.zeros(1, dtype=torch.float64, device=self.device)

        self.running_mean_std = RunningMeanStd(self.obs_dim, self.device) if self.normalize_input else None
        self.value_mean_std = RunningMeanStd(1, self.device) if self.normalize_value else None
        self._amp_input_mean_std = RunningMeanStd(self.amp_obs_dim, self.device) if self._normalize_amp_input else None
        self.running_mean_std_temp = self.running_mean_std.frozen_copy() if self.normalize_input else None

        self._init_buffers()
        self.timer = PhaseTimer(os.environ.get("PHC_PHASE_TIMING", "0") == "1")
        # a simulator backend has to declare that its simulate() is capturable (SyntheticSim does; Isaac Gym's gym.simulate is not)
        self._graph_rollout = (bool(cfg.get("graph_rollout", True)) and os.environ.get("PHC_GRAPH_ROLLOUT", "1") != "0" and
                               bool(getattr(getattr(task, "sim", None), "graph_safe", False)) and
                               self.horizon_length % int(getattr(task.sim, "_body", torch.zeros(1)).shape[0]) == 0)
        self._rollout_graph, self._rollout_out, self._rollout_calls, self._rollout_graph_launches, self._rollout_graph_version = None, None, 0, 0, 0
        self.epoch_num = 0
        self.frame = 0
        self.obs = None
        self.train_result = {}
        self.set_eval()

    # ------------------------------------------------------------------------------------------------------
    # what rl_games hands to an agent (run_hydra.py:199-262, rl_games 1.1.4 a2c_common.A2CBase.__init__)
    # ------------------------------------------------------------------------------------------------------
    @staticmethod
    def _create_vec_env(cfg):
        """rl_games builds the agent from `config['env_name']` / `config['env_config']`: A2CBase creates the vectorised env with
        `vecenv.create_vec_env(env_name, num_actors, **env_config)`, which looks the name up in the registries run_hydra.py fills
        (`vecenv.register('RLGPU', ...)`, `env_configurations.register('rlgpu', {'env_creator': ..., 'vecenv_type': 'RLGPU'})`,
        run_hydra.py:238-240).  The same lookup here: rl_games' registry when the package is importable, else the small registry of
        phc_b200.learning.vecenv_registry (what the tests use).  The result has to expose `.env.task` like the reference's RLGPUEnv."""
        name = cfg.get("env_name")
        if name is None:
            raise KeyError("AMPAgent: config carries neither `vec_env` nor `env_name` (rl_games' params['config']['env_name'])")
        num_actors, env_config = cfg.get("num_actors", 0), dict(cfg.get("env_config", {}) or {})
        from . import vecenv_registry as R
        if name in R.configurations:
            return R.create_vec_env(name, num_actors, **env_config)
        try:
            from rl_games.common import vecenv
        except ImportError:
            raise KeyError(f"AMPAgent: env_name {name!r} is not registered (phc_b200.learning.vecenv_registry.register) and rl_games is not importable")
        return vecenv.create_vec_env(name, num_actors, **env_config)

    @staticmethod
    def _network_spec(net):
        """config['network']: a plain dict (this package, tests) or what rl_games' Runner puts there -- a model object whose builder
        keeps the yaml block (`model.network_builder.params`, rl_games 1.1.4 model_builder.py / network_builder.py).  Returns the dict
        {name, mlp: {units, activation}, disc: {units, activation}, ...} the phc_b200 networks are built from."""
        if isinstance(net, dict):
            return net
        for holder in (net, getattr(net, "network_builder", None), getattr(net, "model", None)):
            p = getattr(holder, "params", None)
            if isinstance(p, dict) and "mlp" in p:
                spec = {"mlp": dict(p["mlp"]), "disc": dict(p.get("disc", p["mlp"])), "name": getattr(holder, "name", p.get("name", "amp"))}
                for k in ("has_softmax", "ending_act", "num_prim", "training_prim"):
                    if k in p:
                        spec[k] = p[k]
                space = p.get("space", {}).get("continuous", {})
                if "sigma_init" in space:
                    spec["sigma_init"] = space["sigma_init"].get("val", -2.9)
                return spec
        raise TypeError("AMPAgent: config['network'] is neither a dict nor an rl_games model / network builder with a `params` block")

    def set_eval(self):
        for r in (self.running_mean_std, self.value_mean_std, self._amp_input_mean_std):
            if r is not None:
                r.eval()

    def set_train(self):
        for r in (self.running_mean_std, self.value_mean_std, self._amp_input_mean_std):
            if r is not None:
                r.train()

    def _init_buffers(self):
        T, N, dev = self.horizon_length, self.num_actors, self.device
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, dtype=dtype, device=dev)
        # rl_games ExperienceBuffer: time-major [T, N, ...]
        self.experience_buffer = {
            "obses": z(T, N, self.obs_dim), "next_obses": z(T, N, self.obs_dim), "rewards": z(T, N, 1),
            "values": z(T, N, 1), "next_values": z(T, N, 1), "dones": z(T, N), "actions": z(T, N, self.actions_num),
            "mus": z(T, N, self.actions_num), "sigmas": z(T, N, self.actions_num), "neglogpacs": z(T, N),
            "amp_obs": z(T, N, self.amp_obs_dim),
        }
        self.tensor_list = ["obses", "next_obses", "actions", "mus", "sigmas", "neglogpacs", "values", "amp_obs"]
        self._amp_obs_demo_buffer = ReplayBuffer(int(self.config["amp_obs_demo_buffer_size"]), self.amp_obs_dim, dev)
        self._amp_replay_buffer = ReplayBuffer(int(self.config["amp_replay_buffer_size"]), self.amp_obs_dim, dev)
        # inference workspaces (rollout batch = N)
        self._x_roll = z(N, self.obs_pad)
        self._val_roll = z(N, 1)
        self._noise = z(N, self.actions_num)
        self._ws_actor_roll = self.engine.workspace("actor_roll", self.model.actor, N)
        self._ws_critic_roll = self.engine.workspace("critic_roll", self.model.critic, N)
        # update workspaces (minibatch B, amp minibatch Bd)
        B, Bd = self.minibatch_size, self._amp_minibatch_size
        self._x_mb = z(B, self.obs_pad)
        self._ws_actor = self.engine.workspace("actor", self.model.actor, B)
        self._ws_critic = self.engine.workspace("critic", self.model.critic, B)
        # The critic is not needed inside the rollout loop: values and next-values enter only GAE, after the last step.  With the
        # grouped GEMM back end they are evaluated afterwards on the stored obses / next_obses, minibatch-sized chunks of both in the
        # same launches (2 x 8 chunks of 16384 rows instead of 2 x 32 batches of 4096 rows).  Row results do not depend on the
        # batching, so this is the same arithmetic (tests/test_gpu_agent.py compares against the per-step path bit for bit).
        self._defer_critic = (self.engine.backend == "tc5s" and bool(self.config.get("deferred_critic", True)) and
                              os.environ.get("PHC_DEFER_CRITIC", "1") != "0")
        if self._defer_critic:
            self._x_mb2 = z(B, self.obs_pad)
            self._ws_critic2 = self.engine.workspace("critic2", self.model.critic, B)
            self._term_steps = z(T, N)
        self._amp_mb = z(3 * Bd, self.amp_pad)           # rows: [agent | replay | demo]
        self._ws_disc = self.engine.workspace("disc", self.model.disc, 3 * Bd)
        du = self.model.disc.hidden
        self._gp_u = [z(Bd, round4(l.out_dim)) for l in du]
        self._gp_e = [z(Bd, round4(l.out_dim)) for l in du]
        self._gp_g = z(Bd, self.amp_pad)
        self._stats = z(16)
        # disc reward over the whole rollout, evaluated in chunks of the amp update batch
        self._ws_disc_r = self.engine.workspace("disc_r", self.model.disc, 3 * Bd)
        self._no_dones = torch.zeros(N, dtype=torch.int64, device=dev)
        self.game_rewards = z(N)
        self.current_rewards = z(N)
        self.current_lengths = z(N)

    # ------------------------------------------------------------------------------------------------------
    # observation / value pre-processing
    # ------------------------------------------------------------------------------------------------------
    def _preproc_obs(self, obs_batch: torch.Tensor, use_temp: bool = False, out: Optional[torch.Tensor] = None,
                     row_idx: Optional[torch.Tensor] = None) -> torch.Tensor:
        """AMPAgent._preproc_obs (amp_agent.py:535-552): normalise with the live or the frozen statistics; with
        use_temp the live statistics are still updated by the batch (train mode)."""
        n = obs_batch.shape[0] if row_idx is None else row_idx.shape[0]
        if out is None:
            out = torch.zeros(n, self.obs_pad, device=self.device)
        if not self.normalize_input:
            src = obs_batch if row_idx is None else obs_batch[row_idx]
            out[:, :self.obs_dim] = src
            return out
        rms = self.running_mean_std_temp if use_temp else self.running_mean_std
        if self.running_mean_std.training and not self.running_mean_std.frozen and n >= 2:
            # normalise with `rms` and fold the RAW rows into the live statistics in the same pass (rows gathered in-kernel)
            self.running_mean_std.apply_update(obs_batch, out, row_idx=row_idx, apply_stats=rms)
        else:
            rms.apply(obs_batch, out, row_idx=row_idx)
        return out

    def _preproc_amp_obs(self, amp_obs: torch.Tensor, out: torch.Tensor, row_idx: Optional[torch.Tensor] = None) -> torch.Tensor:
        if self._normalize_amp_input:
            if self._amp_input_mean_std.training:
                self._amp_input_mean_std.apply_update(amp_obs, out, row_idx=row_idx)
            else:
                self._amp_input_mean_std.apply(amp_obs, out, row_idx=row_idx)
        else:
            out[:, :self.amp_obs_dim] = amp_obs if row_idx is None else amp_obs[row_idx]
        return out

    # ------------------------------------------------------------------------------------------------------
    # rollout
    # ------------------------------------------------------------------------------------------------------
    def get_action_values(self, obs: Dict[str, torch.Tensor], with_value: bool = True) -> Dict[str, torch.Tensor]:
        """CommonAgent.get_action_values (common_agent.py:262-288): normalise, actor + critic forward, sample.
        with_value=False (rollout with the deferred critic): actor only, no "values" entry."""
        N = self.num_actors
        x = self._preproc_obs(obs["obs"], out=self._x_roll)
        val = None
        if not with_value:
            self.engine.forward_group([(self.model.actor, x, self._ws_actor_roll)])
            mu = self._ws_actor_roll["out"]
        elif self.engine.backend == "tc5s":        # actor and critic layer by layer in the same launches
            self.engine.forward_group([(self.model.actor, x, self._ws_actor_roll), (self.model.critic, x, self._ws_critic_roll)])
            mu, val = self._ws_actor_roll["out"], self._ws_critic_roll["out"]
        else:
            mu = self.engine.forward(self.model.actor, x, self._ws_actor_roll)
            val = self.engine.forward(self.model.critic, x, self._ws_critic_roll)
        torch.randn(self._noise.shape, out=self._noise)
        res = {"actions": torch.empty(N, self.actions_num, device=self.device),
               "neglogpacs": torch.empty(N, device=self.device),
               "mus": torch.empty(N, self.actions_num, device=self.device),
               "sigmas": torch.empty(N, self.actions_num, device=self.device)}
        rc = self._lib.phc_gaussian_sample(mu.data_ptr(), mu.stride(0), self.model.sigma.data_ptr(), self._noise.data_ptr(), N,
                                           self.actions_num, res["actions"].data_ptr(), res["neglogpacs"].data_ptr(),
                                           res["mus"].data_ptr(), res["sigmas"].data_ptr(), _stream())
        if rc:
            _lib.check(rc, "phc_gaussian_sample")
        if val is not None:
            res["values"] = self._unnorm_value(val[:, :1])
        return res

    def _rollout_values(self) -> None:
        """values / next_values of the whole rollout from the stored obses / next_obses (see _defer_critic)."""
        eb, critic = self.experience_buffer, self.model.critic
        total, B = self.horizon_length * self.num_actors, self.minibatch_size
        flat = lambda t: t.reshape(total, t.shape[-1])
        o, no, v, nv = flat(eb["obses"]), flat(eb["next_obses"]), flat(eb["values"]), flat(eb["next_values"])
        for s in range(0, total, B):
            n = min(B, total - s)
            x1 = self._preproc_obs(o[s:s + n], out=self._x_mb[:n])
            x2 = self._preproc_obs(no[s:s + n], out=self._x_mb2[:n])
            self.engine.forward_group([(critic, x1, self._ws_critic), (critic, x2, self._ws_critic2)])
            for ws, dst in ((self._ws_critic, v), (self._ws_critic2, nv)):
                if self.normalize_value:
                    self.value_mean_std.apply(ws["out"][:n, :1], dst[s:s + n], unnorm=True)
                else:
                    dst[s:s + n].copy_(ws["out"][:n, :1])
        eb["next_values"].mul_((1.0 - self._term_steps).unsqueeze(-1))

    def _unnorm_value(self, v: torch.Tensor) -> torch.Tensor:
        out = torch.empty(v.shape[0], 1, device=self.device)
        if self.normalize_value:
            self.value_mean_std.apply(v, out, unnorm=True)
        else:
            out.copy_(v)
        return out

    def _eval_critic(self, obs_dict: Dict[str, torch.Tensor]) -> torch.Tensor:
        x = self._preproc_obs(obs_dict["obs"], out=self._x_roll)
        val = self.engine.forward(self.model.critic, x, self._ws_critic_roll)
        return self._unnorm_value(val[:, :1])

    def env_reset(self, env_ids=None):
        return self.vec_env.reset(env_ids)

    def env_step(self, actions):
        obs, rewards, dones, infos = self.vec_env.step(actions)
        return obs, rewards.unsqueeze(1), dones, infos

    def play_steps(self) -> Dict[str, torch.Tensor]:
        """The rollout of one epoch.  The 32 steps are launch-bound when issued one call at a time (~35 short kernels per step
        against ~0.4 ms of GPU work), and nothing in them depends on the host: reset masks instead of index lists, the AMP ring
        head on the device, in-place carried state.  So the first rollout runs eagerly (lazy one-time initialisations), the
        second is captured into ONE CUDA graph and every later one is a single graph launch (`graph_rollout: False` in the
        config or PHC_GRAPH_ROLLOUT=0 keeps the eager loop; the phase timer needs the eager loop too)."""
        if not self._graph_rollout or self.timer.enabled:
            return self._play_steps_eager()
        # the captured launches point at the motion tables and carry _combine_rewards' weights as constants: re-capture when either changes
        version = (getattr(self.vec_env.env.task, "_motion_version", 0), self._task_reward_w, self._disc_reward_w)
        if self._rollout_graph is not None and version != self._rollout_graph_version:
            self._rollout_graph = self._rollout_out = None
            self._rollout_calls = 1
        if self._rollout_graph is not None:
            self._rollout_graph.replay()
            self._lib.phc_launch_count_add(self._rollout_graph_launches)
            return self._rollout_out
        self._rollout_calls += 1
        if self._rollout_calls < 2:
            return self._play_steps_eager()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        l0 = self._lib.phc_launch_count()
        with torch.cuda.graph(g):
            out = self._play_steps_eager()
        self._rollout_graph_launches = self._lib.phc_launch_count() - l0
        self._rollout_graph, self._rollout_out, self._rollout_graph_version = g, out, version
        g.replay()                                   # the capture recorded the work without running it
        return out

    def _play_steps_eager(self) -> Dict[str, torch.Tensor]:
        """AMPAgent.play_steps (amp_agent.py:309-397).  Episode resets are handed to the env as the done MASK of the
        previous step (no nonzero() / host sync on the path)."""
        self.set_eval()
        eb = self.experience_buffer
        terminated_flags = torch.zeros(self.num_actors, device=self.device)
        reward_raw = None
        done_mask = self._no_dones          # the reference starts every rollout with done_indices = [] (amp_agent.py:314)
        T = self.timer
        for n in range(self.horizon_length):
            with T("rollout.env_reset"):
                self.obs = self.env_reset(done_mask)
            with T("rollout.policy"):
                eb["obses"][n].copy_(self.obs["obs"])
                res = self.get_action_values(self.obs, with_value=not self._defer_critic)
                for k in ("actions", "neglogpacs", "values", "mus", "sigmas"):
                    if k in res:
                        eb[k][n].copy_(res[k])
            with T("rollout.env_step"):
                self.obs, rewards, self.dones, infos = self.env_step(res["actions"])
            with T("rollout.store"):
                eb["rewards"][n].copy_(rewards)
                eb["next_obses"][n].copy_(self.obs["obs"])
                eb["dones"][n].copy_(self.dones)
                if "amp_obs_export" in infos:
                    infos["amp_obs_export"](eb["amp_obs"][n])            # AMP ring -> newest-first window, written in place
                else:
                    eb["amp_obs"][n].copy_(infos["amp_obs"])
                terminated = infos["terminate"].float()
                terminated_flags += terminated
                rr = infos["reward_raw"].mean(dim=0)
                reward_raw = rr if reward_raw is None else reward_raw + rr
            with T("rollout.critic_next"):
                if self._defer_critic:
                    self._term_steps[n].copy_(terminated)
                else:
                    next_vals = self._eval_critic(self.obs)
                    next_vals *= (1.0 - terminated.unsqueeze(-1))
                    eb["next_values"][n].copy_(next_vals)
            not_dones = 1.0 - self.dones.float()
            self.current_rewards.add_(rewards.squeeze(1)).mul_(not_dones)      # in place: state carried across (graph-replayed) rollouts
            self.current_lengths.add_(1).mul_(not_dones)
            done_mask = self.dones

        if self._defer_critic:
            with T("rollout.critic_batched"):
                self._rollout_values()
        mb_fdones = eb["dones"]
        with T("rollout.disc_reward"):
            amp_rewards = self._calc_amp_rewards(eb["amp_obs"])
            mb_rewards = self._combine_rewards(eb["rewards"], amp_rewards)
        with T("rollout.gae"):
            mb_advs = self.discount_values(mb_fdones, eb["values"], mb_rewards, eb["next_values"])
        mb_returns = self._last_returns
        flat = lambda t: t.transpose(0, 1).reshape(self.batch_size, *t.shape[2:])      # swap_and_flatten01
        batch_dict = {k: flat(eb[k]) for k in self.tensor_list}
        batch_dict["returns"] = flat(mb_returns)
        batch_dict["terminated_flags"] = terminated_flags
        batch_dict["reward_raw"] = reward_raw / self.horizon_length
        batch_dict["played_frames"] = self.batch_size
        batch_dict["disc_rewards"] = flat(amp_rewards["disc_rewards"])
        batch_dict["mb_rewards"] = flat(mb_rewards)
        batch_dict["mb_advs"] = flat(mb_advs)
        return batch_dict

    # ------------------------------------------------------------------------------------------------------
    # rewards / GAE / advantages
    # ------------------------------------------------------------------------------------------------------
    def _calc_amp_rewards(self, amp_obs: torch.Tensor) -> Dict[str, torch.Tensor]:
        """AMPAgent._calc_amp_rewards / _calc_disc_rewards (amp_agent.py:859-878) over the whole rollout."""
        flat = amp_obs.reshape(-1, self.amp_obs_dim)
        total = flat.shape[0]
        disc_r = torch.empty(total, device=self.device)
        chunk = self._amp_mb.shape[0]
        for s in range(0, total, chunk):
            n = min(chunk, total - s)
            if self._normalize_amp_input:
                self._amp_input_mean_std.apply(flat[s:s + n], self._amp_mb, n=n)
            else:
                self._amp_mb[:n, :self.amp_obs_dim].copy_(flat[s:s + n])
            logits = self.engine.forward(self.model.disc, self._amp_mb, self._ws_disc_r)
            rc = self._lib.phc_disc_reward(logits.data_ptr(), logits.stride(0), None, n, self._disc_reward_scale, 0.0, 0.0,
                                           disc_r[s:].data_ptr(), None, _stream())
            if rc:
                _lib.check(rc, "phc_disc_reward")
        return {"disc_rewards": disc_r.view(*amp_obs.shape[:-1], 1)}

    def _combine_rewards(self, task_rewards: torch.Tensor, amp_rewards: Dict[str, torch.Tensor]) -> torch.Tensor:
        return self._task_reward_w * task_rewards + self._disc_reward_w * amp_rewards["disc_rewards"]

    def discount_values(self, mb_fdones, mb_values, mb_rewards, mb_next_values) -> torch.Tensor:
        """CommonAgent.discount_values (common_agent.py:493-505) -> phc_gae (also keeps returns = advs + values)."""
        advs, rets = ops.gae(mb_fdones.float().contiguous(), mb_values.contiguous(), mb_rewards.contiguous(),
                             mb_next_values.contiguous(), self.gamma, self.tau)
        self._last_returns = rets
        return advs

    def _calc_advs(self, batch_dict) -> torch.Tensor:
        return ops.adv_norm(batch_dict["returns"].contiguous(), batch_dict["values"].contiguous(), self.normalize_advantage)

    def prepare_dataset(self, batch_dict) -> Dict[str, torch.Tensor]:
        """CommonAgent.prepare_dataset (:357-398) + AMPAgent.prepare_dataset (amp_agent.py:399-411)."""
        advantages = self._calc_advs(batch_dict)
        values, returns = batch_dict["values"], batch_dict["returns"]
        if self.normalize_value:
            values, returns = self.value_mean_std(values), self.value_mean_std(returns)
        self.dataset = dict(old_values=values, old_logp_actions=batch_dict["neglogpacs"], advantages=advantages,
                            returns=returns, actions=batch_dict["actions"], obs=batch_dict["obses"], mu=batch_dict["mus"],
                            sigma=batch_dict["sigmas"], amp_obs=batch_dict["amp_obs"],
                            amp_obs_demo_idx=batch_dict["amp_obs_demo_idx"], amp_obs_replay_idx=batch_dict["amp_obs_replay_idx"])
        self._idx_buf = torch.randperm(self.batch_size, device=self.device)
        return self.dataset

    # ------------------------------------------------------------------------------------------------------
    # update
    # ------------------------------------------------------------------------------------------------------
    def calc_gradients(self, input_dict: Dict[str, torch.Tensor]) -> None:
        """One PPO/AMP minibatch: forward, losses, backward into the flat gradient bucket, all-reduce, clip, Adam.
        input_dict carries `idx` (rows of the epoch dataset) instead of materialised copies of the big tensors
        (AMPDataset._get_item gathers ~0.5 GB per minibatch of which 3/4 of the AMP rows are dropped afterwards).
        train_epoch runs the same three stages software-pipelined (see _minibatch_pipeline)."""
        idx = input_dict["idx"]
        prepared = self._prepare_minibatch(idx) if self.engine.backend == "tc5s" else None
        self._compute_gradients(idx, prepared)
        scale = self._reducer.begin(self.model.grads) if self.multi_gpu else 1.0
        if self.multi_gpu:
            self._reducer.end()
        self._optimizer_step(scale)

    def _prepare_minibatch(self, idx: torch.Tensor):
        """Everything of a minibatch that does not depend on the weights: gather + normalise the observation and the three AMP row
        blocks into the update workspaces (and fold the batch into the running statistics, as RunningMeanStd.forward does in train
        mode).  Split off so that train_epoch can issue it for minibatch i + 1 while the gradient all-reduce of minibatch i runs."""
        self.set_train()
        ds, T = self.dataset, self.timer
        Bd = self._amp_minibatch_size
        with T("update.preproc_obs"):
            x = self._preproc_obs(ds["obs"], use_temp=self.temp_running_mean, out=self._x_mb, row_idx=idx)
        with T("update.disc_preproc"):
            aidx = idx[:Bd]
            xa = self._amp_mb
            self._preproc_amp_obs(ds["amp_obs"], xa[0:Bd], row_idx=aidx)
            self._preproc_amp_obs(self._amp_replay_src, xa[Bd:2 * Bd], row_idx=ds["amp_obs_replay_idx"][aidx])
            self._preproc_amp_obs(self._amp_obs_demo_buffer.data, xa[2 * Bd:3 * Bd], row_idx=ds["amp_obs_demo_idx"][aidx])
        return x, xa

    def _compute_gradients(self, idx: torch.Tensor, prepared=None) -> None:
        self.set_train()
        net, eng, ds = self.model, self.engine, self.dataset
        B, Bd, A = idx.shape[0], self._amp_minibatch_size, self.actions_num
        inv_b = 1.0 / B
        st = _stream()
        self._stats.zero_()
        net.grads.zero_()
        if eng.backend == "tc5s":
            x, xa = prepared if prepared is not None else self._prepare_minibatch(idx)
            self._grouped_core(x, xa, Bd, st, lambda: self._loss_grads(ds, idx, B, Bd, A, inv_b, st, self._ws_actor["out"], self._ws_critic["out"],
                                                                       self._ws_disc["out"]))
        else:
            self._update_sequential(ds, idx, B, Bd, A, inv_b, st)
        self._last_B, self._last_Bd = B, Bd

    def _optimizer_step(self, grad_scale: float) -> None:
        lib, net, st = self._lib, self.model, _stream()
        with self.timer("update.optim"):
            self.opt_step += 1
            _lib.check(lib.phc_grad_sumsq(net.grads.data_ptr(), net.num_floats, self._gsumsq.data_ptr(), st))
            _lib.check(lib.phc_adam_step(net.params.data_ptr(), net.grads.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(),
                                         net.num_floats, self._gsumsq.data_ptr(), grad_scale,
                                         self.grad_norm if self.truncate_grads else 0.0, self.last_lr, 0.9, 0.999, 1e-8,
                                         self.opt_step, st))
            if self.engine.uses_images:
                net.refresh_images()
            if self.engine.backend == "tc5":
                net.refresh_split()                    # hi/lo operand copies of the updated weights

    def _minibatch_pipeline(self) -> None:
        """The mini_epochs x num_minibatches updates of an epoch (amp_agent.py:460-483), software-pipelined: the gradient
        all-reduce of minibatch i is issued on a side stream and, while it runs over NVLink, the compute stream already gathers
        and normalises the rows of minibatch i + 1 (weight-independent, ~0.3 ms); Adam(i) follows once the reduced bucket is
        back.  The collective leaves the critical path without splitting the single flat all-reduce per minibatch."""
        mb = self.minibatch_size
        grouped = self.engine.backend == "tc5s"

        def indices():
            for _ in range(self.mini_epochs_num):
                for i in range(self.num_minibatches):
                    yield self._idx_buf[i * mb:(i + 1) * mb]
                self._idx_buf = torch.randperm(self.batch_size, device=self.device)
        it = indices()
        idx = next(it, None)
        prepared = self._prepare_minibatch(idx) if (grouped and idx is not None) else None
        while idx is not None:
            self._compute_gradients(idx, prepared)
            scale = self._reducer.begin(self.model.grads) if self.multi_gpu else 1.0
            idx = next(it, None)                       # (a new permutation is drawn here at mini-epoch boundaries)
            prepared = self._prepare_minibatch(idx) if (grouped and idx is not None) else None
            if self.multi_gpu:
                self._reducer.end()
            self._optimizer_step(scale)

    def _update_sequential(self, ds, idx, B, Bd, A, inv_b, st) -> None:
        """Forward / losses / backward one network after the other, one launch per GEMM (mma.sync and pre-split wgmma back ends)."""
        lib, net, eng, T = self._lib, self.model, self.engine, self.timer
        # ---- actor / critic ----------------------------------------------------------------------------------
        with T("update.preproc_obs"):
            x = self._preproc_obs(ds["obs"], use_temp=self.temp_running_mean, out=self._x_mb, row_idx=idx)
        with T("update.ac_forward"):
            mu = eng.forward(net.actor, x, self._ws_actor)
            val = eng.forward(net.critic, x, self._ws_critic)
        with T("update.ac_loss"):
            actions, old_nlp, adv = ds["actions"][idx], ds["old_logp_actions"][idx], ds["advantages"][idx]
            old_mu, old_sigma, rets = ds["mu"][idx], ds["sigma"][idx], ds["returns"][idx].reshape(-1)
            dmu, dv = self._ws_actor["dout"], self._ws_critic["dout"]
            _lib.check(lib.phc_ppo_actor_grad(mu.data_ptr(), mu.stride(0), net.sigma.data_ptr(), actions.data_ptr(), old_nlp.data_ptr(),
                                              adv.data_ptr(), old_mu.data_ptr(), old_sigma.data_ptr(), B, A, self.e_clip,
                                              self.bounds_loss_coef, inv_b, dmu.data_ptr(), dmu.stride(0), self._stats.data_ptr(), st))
            _lib.check(lib.phc_ppo_critic_grad(val.data_ptr(), val.stride(0), rets.data_ptr(), B, self.critic_coef, inv_b,
                                               dv.data_ptr(), dv.stride(0), self._stats.data_ptr(), st))
        with T("update.ac_backward"):
            eng.backward(net.actor, x, self._ws_actor)
            eng.backward(net.critic, x, self._ws_critic)

        # ---- discriminator: rows [agent | replay | demo] of the first Bd minibatch samples ---------------------
        with T("update.disc_preproc"):
            aidx = idx[:Bd]
            xa = self._amp_mb
            self._preproc_amp_obs(ds["amp_obs"], xa[0:Bd], row_idx=aidx)
            self._preproc_amp_obs(self._amp_replay_src, xa[Bd:2 * Bd], row_idx=ds["amp_obs_replay_idx"][aidx])
            self._preproc_amp_obs(self._amp_obs_demo_buffer.data, xa[2 * Bd:3 * Bd], row_idx=ds["amp_obs_demo_idx"][aidx])
        with T("update.disc_forward"):
            logits = eng.forward(net.disc, xa, self._ws_disc)
        with T("update.disc_backward"):
            dl = self._ws_disc["dout"]
            _lib.check(lib.phc_disc_logit_grad(logits.data_ptr(), logits.stride(0), 2 * Bd, Bd, self._disc_coef, dl.data_ptr(),
                                               dl.stride(0), self._stats.data_ptr(), st))
            eng.backward(net.disc, xa, self._ws_disc)
        with T("update.disc_grad_penalty"):
            self._disc_grad_penalty_backward(xa[2 * Bd:3 * Bd], [h[2 * Bd:3 * Bd] for h in self._ws_disc["h"]], Bd)
            # logit regulariser and weight decay (amp_agent.py:745-747, :771-775): d/dW (c * sum W^2) = 2 c W
            head = net.disc.head
            _lib.check(lib.phc_axpy2d(net.weight(head).data_ptr(), head.in_pad, net.weight(head, True).data_ptr(), head.in_pad, 1,
                                      head.in_dim, 2.0 * self._disc_coef * self._disc_logit_reg, self._stats[11:].data_ptr(), st))
            if self._disc_weight_decay != 0:
                for l in net.disc.layers:
                    _lib.check(lib.phc_axpy2d(net.weight(l).data_ptr(), l.in_pad, net.weight(l, True).data_ptr(), l.in_pad, l.out_dim,
                                              l.in_dim, 2.0 * self._disc_coef * self._disc_weight_decay, self._stats[12:].data_ptr(), st))


    def _loss_grads(self, ds, idx, B, Bd, A, inv_b, st, mu, val, logits) -> None:
        """d loss / d (mu, value, logit) of the minibatch `idx`: the dataset arrays are addressed through idx inside the kernels."""
        lib, net = self._lib, self.model
        dmu, dv, dl = self._ws_actor["dout"], self._ws_critic["dout"], self._ws_disc["dout"]
        arr = [ds[k] if ds[k].is_contiguous() else ds[k].contiguous() for k in ("actions", "old_logp_actions", "advantages", "mu", "sigma", "returns")]
        for k, t in zip(("actions", "old_logp_actions", "advantages", "mu", "sigma", "returns"), arr):
            ds[k] = t                                    # (flattened views of the experience buffer are made contiguous once per epoch)
        _lib.check(lib.phc_ppo_grads_gather(mu.data_ptr(), mu.stride(0), net.sigma.data_ptr(), arr[0].data_ptr(), arr[1].data_ptr(), arr[2].data_ptr(),
                                            arr[3].data_ptr(), arr[4].data_ptr(), val.data_ptr(), val.stride(0), arr[5].data_ptr(), idx.data_ptr(), B, A,
                                            self.e_clip, self.bounds_loss_coef, self.critic_coef, inv_b, dmu.data_ptr(), dmu.stride(0), dv.data_ptr(),
                                            dv.stride(0), self._stats.data_ptr(), st), "phc_ppo_grads_gather")
        _lib.check(lib.phc_disc_logit_grad(logits.data_ptr(), logits.stride(0), 2 * Bd, Bd, self._disc_coef, dl.data_ptr(),
                                           dl.stride(0), self._stats.data_ptr(), st))

    def _grouped_core(self, x, xa, Bd, st, loss_fn) -> None:
        """The minibatch with the grouped GEMM (phc_gemm_group): actor, critic and discriminator advance layer by layer TOGETHER --
        one persistent launch per layer index forward (3 problems), one per layer index backward (dW and dX of the three networks
        plus the step of the gradient-penalty chain that is ready: up to 8 problems) -- instead of ~30 separate GEMM launches whose
        tile counts each leave a partial last wave on the 132 SMs.
        forward (grouped) -> loss_fn() writes d loss / d outputs into the workspaces' `dout` -> backward (grouped, with the
        gradient-penalty chain merged in) -> discriminator regularisers.  x / xa are the normalised, zero-padded inputs."""
        lib, net, eng, T = self._lib, self.model, self.engine, self.timer
        stacks = [(net.actor, x, self._ws_actor), (net.critic, x, self._ws_critic), (net.disc, xa, self._ws_disc)]
        with T("update.forward"):
            eng.forward_group(stacks)
        with T("update.losses"):
            loss_fn()
            for stk, _, ws in stacks:
                if stk.head_relu:                       # MCP composer: activation after the head
                    silu = stk.activation == "silu"
                    aux = ws["z_out"] if silu else ws["out"]
                    _lib.check(lib.phc_act_backward(ws["dout"].data_ptr(), ws["dout"].stride(0), aux.data_ptr(), aux.stride(0), ws["dout"].shape[0],
                                                    stk.out_dim, _lib.PHC_ACT_SILU if silu else _lib.PHC_ACT_RELU, st))
        with T("update.backward"):
            gp = self._gp_steps(xa[2 * Bd:3 * Bd], Bd, st)
            depth = max(len(stk.layers) for stk, _, _ in stacks)
            for k in range(max(depth, len(gp))):
                descs, sums = [], []
                for stk, xin, ws in stacks:
                    li = len(stk.layers) - 1 - k
                    if li >= 0:
                        dw, dx = eng.bwd_descs(stk, li, xin, ws)
                        descs += [dw, dx]
                        l = stk.layers[li]
                        dY = ws["dout"] if li == len(stk.layers) - 1 else ws["dh"][li]
                        sums.append((dY, dY.shape[0], l.out_dim, net.bias(l, grad=True)))
                after = None
                if k < len(gp):
                    gdescs, after = gp[k]
                    descs += gdescs
                eng.run_group(descs)
                eng.colsum_group(sums)
                if after is not None:
                    after()
            head = net.disc.head
            _lib.check(lib.phc_axpy2d(net.weight(head).data_ptr(), head.in_pad, net.weight(head, True).data_ptr(), head.in_pad, 1,
                                      head.in_dim, 2.0 * self._disc_coef * self._disc_logit_reg, self._stats[11:].data_ptr(), st))
            if self._disc_weight_decay != 0:
                for l in net.disc.layers:
                    _lib.check(lib.phc_axpy2d(net.weight(l).data_ptr(), l.in_pad, net.weight(l, True).data_ptr(), l.in_pad, l.out_dim,
                                              l.in_dim, 2.0 * self._disc_coef * self._disc_weight_decay, self._stats[12:].data_ptr(), st))

    def _gp_steps(self, x_demo: torch.Tensor, Bd: int, st):
        """The gradient-penalty chain of _disc_grad_penalty_backward as a list of steps [(problems, after-hook)] that
        _update_grouped merges into its per-layer launches: L input-gradient GEMMs down to g = d logit / d x, the penalty
        itself (phc_scale_sumsq), then per layer the weight-gradient and the forward-form GEMM of the backward chain."""
        lib, net, eng = self._lib, self.model, self.engine
        hid, head = net.disc.hidden, net.disc.head
        L = len(hid)
        ws = self._ws_disc
        h_demo = [h[2 * Bd:3 * Bd] for h in ws["h"]]
        bits = [hb[2 * Bd:3 * Bd] for hb in ws["hbits"]] if "hbits" in ws else None
        mask = lambda i: dict(act=_lib.PHC_ACT_MASK_BITS, aux=bits[i]) if bits is not None else dict(aux=h_demo[i])
        u, e, g = self._gp_u, self._gp_e, self._gp_g
        _lib.check(lib.phc_relu_mask_row(h_demo[L - 1].data_ptr(), h_demo[L - 1].stride(0), net.weight(head).data_ptr(), Bd,
                                         hid[L - 1].out_dim, u[L - 1].data_ptr(), u[L - 1].stride(0), st))
        steps = []
        for li in range(L - 1, 0, -1):
            l = hid[li]
            steps.append(([eng.gdesc(u[li], True, net.weight(l), False, u[li - 1], Bd, l.in_dim, l.out_dim, B_img=eng.image(l, False),
                                     **mask(li - 1))], None))
        l0 = hid[0]
        c = self._disc_coef * self._disc_grad_penalty

        def penalty():
            _lib.check(lib.phc_scale_sumsq(g.data_ptr(), g.stride(0), Bd, l0.in_dim, 2.0 * c / Bd, self._stats[10:].data_ptr(), st))
        steps.append(([eng.gdesc(u[0], True, net.weight(l0), False, g, Bd, l0.in_dim, l0.out_dim, B_img=eng.image(l0, False))], penalty))
        for li in range(L):
            l = hid[li]
            src = g if li == 0 else e[li - 1]
            after = None
            if li == L - 1:
                after = lambda: eng.colsum(e[L - 1], Bd, hid[L - 1].out_dim, net.weight(head, True))
            steps.append(([eng.dw_desc(u[li], src, net.weight(l, True), l.out_dim, l.in_dim, Bd),
                           eng.gdesc(src, True, net.weight(l), True, e[li], Bd, l.out_dim, l.in_dim, B_img=eng.image(l, True), **mask(li))],
                          after))
        return steps

    def _disc_grad_penalty_backward(self, x_demo: torch.Tensor, h_demo, Bd: int) -> None:
        """Gradient penalty 5 * mean_b ||d logit_b / d x_b||^2 on the demo rows (amp_agent.py:749-768), hand-derived for
        the ReLU MLP (the reference uses autograd.grad(create_graph=True)):
            u_L = relu'(z_L) * w_head ; u_{l-1} = relu'(z_{l-1}) * (u_l W_l) ; g = u_1 W_1
            P = c/B sum ||g||^2 ; dP/dg = 2c/B g ; dP/dW_1 += u_1^T dg ; e_1 = relu'(z_1) * (dg W_1^T) ;
            dP/dW_l += u_{l-1}^T e_{l-1}... ; dP/dw_head += colsum(relu'(z_L) * (e W^T))
        second derivatives of ReLU vanish, so the masks are constants."""
        lib, net, eng, st = self._lib, self.model, self.engine, _stream()
        hid = net.disc.hidden
        L = len(hid)
        head = net.disc.head
        u, e = self._gp_u, self._gp_e
        # forward of the input-gradient: top mask times the head weights, then down through the layers
        _lib.check(lib.phc_relu_mask_row(h_demo[L - 1].data_ptr(), h_demo[L - 1].stride(0), net.weight(head).data_ptr(), Bd,
                                         hid[L - 1].out_dim, u[L - 1].data_ptr(), u[L - 1].stride(0), st))
        for li in range(L - 1, 0, -1):
            l = hid[li]
            eng.gemm(u[li], True, net.weight(l), False, u[li - 1], Bd, l.in_dim, l.out_dim, mask=h_demo[li - 1])
        l0 = hid[0]
        eng.gemm(u[0], True, net.weight(l0), False, self._gp_g, Bd, l0.in_dim, l0.out_dim)
        c = self._disc_coef * self._disc_grad_penalty
        _lib.check(lib.phc_scale_sumsq(self._gp_g.data_ptr(), self._gp_g.stride(0), Bd, l0.in_dim, 2.0 * c / Bd,
                                       self._stats[10:].data_ptr(), st))
        # backward of that chain
        tiles = lambda l: ((l.out_dim + 127) // 128) * ((l.in_dim + 127) // 128)
        from .networks import _splits
        eng.gemm(u[0], False, self._gp_g, False, net.weight(l0, True), l0.out_dim, l0.in_dim, Bd, accumulate=True,
                 k_splits=_splits(tiles(l0), Bd))
        eng.gemm(self._gp_g, True, net.weight(l0), True, e[0], Bd, l0.out_dim, l0.in_dim, mask=h_demo[0])
        for li in range(1, L):
            l = hid[li]
            eng.gemm(u[li], False, e[li - 1], False, net.weight(l, True), l.out_dim, l.in_dim, Bd, accumulate=True,
                     k_splits=_splits(tiles(l), Bd))
            eng.gemm(e[li - 1], True, net.weight(l), True, e[li], Bd, l.out_dim, l.in_dim, mask=h_demo[li])
        eng.colsum(e[L - 1], Bd, hid[L - 1].out_dim, net.weight(head, True))

    def train_result_dict(self) -> Dict[str, float]:
        """Scalars of the last minibatch (one device->host read; call outside the timed path)."""
        s = self._stats.tolist()
        B, Bd = self._last_B, self._last_Bd
        return dict(actor_loss=s[0] / B, b_loss=s[1] / B, actor_clip_frac=s[2] / B, kl=s[3] / B, entropy=s[4] / B,
                    critic_loss=s[5] / B, disc_loss_agent=s[6] / (2 * Bd), disc_loss_demo=s[7] / Bd,
                    disc_agent_acc=s[8] / (2 * Bd), disc_demo_acc=s[9] / Bd, disc_grad_penalty=s[10] / Bd,
                    disc_logit_loss=s[11])

    def _disc_loss(self, disc_agent_logit=None, disc_demo_logit=None, obs_demo=None) -> Dict[str, float]:
        """AMPAgent._disc_loss (amp_agent.py:732-789).  The loss and its gradient (incl. the gradient penalty) are produced
        inside calc_gradients by phc_disc_logit_grad + the GEMM chain; this returns the reference's info dict for the LAST
        minibatch from the statistics those kernels accumulated (arguments are accepted for signature parity and ignored)."""
        r = self.train_result_dict()
        bce = 0.5 * (r["disc_loss_agent"] + r["disc_loss_demo"])
        wd = 0.0
        if self._disc_weight_decay != 0:
            wd = self._disc_weight_decay * float(sum((self.model.weight(l)[:, :l.in_dim] ** 2).sum() for l in self.model.disc.layers))
        total = bce + self._disc_logit_reg * r["disc_logit_loss"] + self._disc_grad_penalty * r["disc_grad_penalty"] + wd
        return dict(disc_loss=total, disc_grad_penalty=r["disc_grad_penalty"], disc_logit_loss=r["disc_logit_loss"],
                    disc_agent_acc=r["disc_agent_acc"], disc_demo_acc=r["disc_demo_acc"])

    def eval(self) -> Dict[str, float]:
        """CommonAgent.eval (common_agent.py:187-189): nothing to evaluate at this level; IMAmpAgent (im_amp.py) overrides it."""
        return {}

    def pre_epoch(self, epoch_num: int) -> None:
        task = self.vec_env.env.task
        # AMPAgent.pre_epoch (amp_agent.py:506-516): a new set of clips every shape_resampling_interval epochs ("+ 1 to evade the evaluations")
        if (getattr(task, "humanoid_type", "") in ("smpl", "smplh", "smplx") and hasattr(getattr(task, "_motion_data", None), "load_motions")
                and hasattr(task.sim, "skeleton_trees") and epoch_num > 1 and epoch_num % int(task.shape_resampling_interval) == 1):
            task.resample_motions()
        # the get-up schedule (amp_agent.py:518-525): fall starts only and the discriminator reward alone until getup_udpate_epoch
        if getattr(task, "humanoid_type", "") in ("smpl", "smplh", "smplx") and getattr(task, "getup_schedule", False):
            task.update_getup_schedule(epoch_num, getup_udpate_epoch=task.getup_udpate_epoch)
            if epoch_num > task.getup_udpate_epoch:
                self._task_reward_w, self._disc_reward_w = 0.5, 0.5
            else:
                self._task_reward_w, self._disc_reward_w = 0, 1
        if self.normalize_input:
            self.running_mean_std_temp = self.running_mean_std.frozen_copy()   # amp_agent.py:527-528

    def post_epoch(self, epoch_num: int) -> None:
        if self.multi_gpu:          # hvd.sync_stats (common_agent.py:126-127)
            D.sync_running_stats([self.running_mean_std, self.value_mean_std, self._amp_input_mean_std])
        if self.normalize_input:
            self.running_mean_std_temp = self.running_mean_std.frozen_copy()

    def _update_amp_demos(self) -> None:
        self._amp_obs_demo_buffer.store(self.vec_env.env.fetch_amp_obs_demo(self._amp_batch_size))

    def _init_amp_demo_buf(self) -> None:
        size = self._amp_obs_demo_buffer.get_buffer_size()
        for _ in range((size + self._amp_batch_size - 1) // self._amp_batch_size):
            self._update_amp_demos()

    def _store_replay_amp_obs(self, amp_obs: torch.Tensor) -> None:
        """amp_agent.py:880-894."""
        buf = self._amp_replay_buffer
        if buf.get_total_count() > buf.get_buffer_size():
            keep = torch.rand(amp_obs.shape[0], device=self.device) < self._amp_replay_keep_prob
            amp_obs = amp_obs[keep]
        if amp_obs.shape[0] > buf.get_buffer_size():
            amp_obs = amp_obs[torch.randperm(amp_obs.shape[0], device=self.device)[:buf.get_buffer_size()]]
        buf.store(amp_obs)

    def train_epoch(self) -> Dict[str, torch.Tensor]:
        """AMPAgent.train_epoch (amp_agent.py:413-504)."""
        self.pre_epoch(self.epoch_num)
        t0 = time.time()
        batch_dict = self.play_steps()
        t1 = time.time()
        _prep = self.timer("epoch.prepare")
        _prep.__enter__()
        self._update_amp_demos()
        n = batch_dict["amp_obs"].shape[0]
        batch_dict["amp_obs_demo_idx"] = self._amp_obs_demo_buffer.sample_indices(n)
        if self._amp_replay_buffer.get_total_count() == 0:
            self._amp_replay_src = batch_dict["amp_obs"]
            batch_dict["amp_obs_replay_idx"] = torch.arange(n, device=self.device)
        else:
            self._amp_replay_src = self._amp_replay_buffer.data
            batch_dict["amp_obs_replay_idx"] = self._amp_replay_buffer.sample_indices(n)
        self.set_train()
        self.prepare_dataset(batch_dict)
        _prep.__exit__()
        self._minibatch_pipeline()
        with self.timer("epoch.replay_store"):
            self._store_replay_amp_obs(batch_dict["amp_obs"])
        self.post_epoch(self.epoch_num)
        t2 = time.time()
        self.epoch_num += 1
        self.frame += self.batch_size * self.world
        return dict(play_time=t1 - t0, update_time=t2 - t1, total_time=t2 - t0, terminated_flags=batch_dict["terminated_flags"],
                    reward_raw=batch_dict["reward_raw"], mb_rewards=batch_dict["mb_rewards"], returns=batch_dict["returns"],
                    disc_rewards=batch_dict["disc_rewards"])

    def train(self, max_epochs: Optional[int] = None):
        """CommonAgent.train (common_agent.py:100-185) without the logging / checkpoint cadence side channels."""
        self.obs = self.env_reset()
        self._init_amp_demo_buf()
        max_epochs = self.config["max_epochs"] if max_epochs is None else max_epochs
        info = None
        while self.epoch_num < max_epochs:
            info = self.train_epoch()
        return info

    # ------------------------------------------------------------------------------------------------------
    # checkpoint dict, same keys as the reference (amp_agent.py:69-102,:158-166; SURVEY.md section 5)
    # ------------------------------------------------------------------------------------------------------
    def get_stats_weights(self) -> Dict:
        st = {}
        if self.normalize_input:
            st["running_mean_std"] = self.running_mean_std.state_dict()
        if self.normalize_value:
            st["reward_mean_std"] = self.value_mean_std.state_dict()
        if self._normalize_amp_input:
            st["amp_input_mean_std"] = self._amp_input_mean_std.state_dict()
        return st

    def set_stats_weights(self, weights: Dict) -> None:
        if self.normalize_input and "running_mean_std" in weights:
            self.running_mean_std.load_state_dict(weights["running_mean_std"])
            self.running_mean_std_temp = self.running_mean_std.frozen_copy()
        if self.normalize_value and "reward_mean_std" in weights:
            self.value_mean_std.load_state_dict(weights["reward_mean_std"])
        if self._normalize_amp_input and "amp_input_mean_std" in weights:
            self._amp_input_mean_std.load_state_dict(weights["amp_input_mean_std"])

    def get_full_state_weights(self) -> Dict:
        state = {"model": self.model.state_dict(), "epoch": self.epoch_num, "frame": self.frame,
                 "optimizer": {"exp_avg": self.exp_avg.clone(), "exp_avg_sq": self.exp_avg_sq.clone(), "step": self.opt_step},
                 "last_mean_rewards": 0}
        state.update(self.get_stats_weights())
        return state

    def set_full_state_weights(self, weights: Dict) -> None:
        self.model.load_state_dict(weights["model"])
        if self.engine.backend == "tc5":
            self.model.refresh_split()
        self.epoch_num = weights.get("epoch", 0)
        self.frame = weights.get("frame", 0)
        opt = weights.get("optimizer")
        if isinstance(opt, dict) and "exp_avg" in opt:
            self.exp_avg.copy_(opt["exp_avg"].to(self.device))
            self.exp_avg_sq.copy_(opt["exp_avg_sq"].to(self.device))
            self.opt_step = int(opt["step"])
        self.set_stats_weights(weights)

    def save(self, fn: str) -> None:
        torch.save(self.get_full_state_weights(), fn if fn.endswith(".pth") else fn + ".pth")

    def restore(self, fn: str) -> None:
        self.set_full_state_weights(torch.load(fn, map_location=self.device, weights_only=False))
