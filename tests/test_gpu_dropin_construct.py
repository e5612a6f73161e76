"""The construction path of the reference's entry point, on the phc_b200 classes (VERDICT r1 "make the drop-in real"):

  parse_task.py:60     task = eval(args.task)(cfg=cfg, sim_params=..., physics_engine=..., device_type=..., device_id=..., headless=...)
  run_hydra.py:199-262 rl_games builds the agent from params['config'] (env_name / env_config / num_actors / network builder)
  im_amp.py:37-39      class IMAmpAgent(amp_agent.AMPAgent): __init__(self, base_name, config): super().__init__(base_name, config)

with a fake simulator side standing in for Isaac Gym (the reference's original task class is what phc_b200.dropin registers as the
backend factory; here a factory returns a synthetic owner of the same tensors + asset data): the task is built from the hydra-shaped
cfg tree with NO motion_data (MotionLibSMPL loads env.motion_file itself), the agent from the rl_games-shaped config, one epoch
trains, resample_motions() loads a different set of clips on the device and keeps every humanoid in place."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from phc_b200 import synthetic as syn
from phc_b200.env import backends
from phc_b200.env.humanoid_im import HumanoidIm, SyntheticSim, VecTaskPythonWrapper
from phc_b200.learning import vecenv_registry as R
from phc_b200.learning.amp_agent import AMPAgent
from tests.test_gpu_motion_load import _random_clips

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N, J = 48, 24


class FakeGymOwner(SyntheticSim):
    """What phc_b200.env.backends documents: state tensors + simulate + set_env_state + the per-env asset data of Humanoid."""
    graph_safe = False          # like Isaac Gym: simulate() is not a CUDA-stream operation, the rollout stays an eager loop

    def __init__(self, num_envs, device):
        m = syn.make_motions(8, seed=1, min_frames=20, max_frames=30)
        super().__init__(m, num_envs, device, seed=3)
        rng = np.random.default_rng(0)
        off = rng.standard_normal((J, 3)) * 0.15
        off[0] = 0
        self.skeleton_trees = [SimpleNamespace(local_translation=off, parent_indices=np.array(syn.SMPL_PARENTS, dtype=np.int32),
                                               node_names=[f"b{j}" for j in range(J)]) for _ in range(num_envs)]
        self.humanoid_shapes = torch.zeros(num_envs, 17)
        self.humanoid_limb_and_weights = torch.zeros(num_envs, 10)
        self.pd_action_offset = torch.zeros(3 * (J - 1))
        self.pd_action_scale = torch.full((3 * (J - 1),), 1.5)
        self.applied = 0

    def set_env_state(self, mask, rigid_body_state, dof_state):
        self.applied += 1


def _clip_file(M, seed):
    z = _random_clips(M, J, seed=seed, min_f=30, max_f=70)
    clips, s = {}, 0
    for i, n in enumerate(z["num_frames"]):
        clips[f"clip{i}"] = {"pose_quat_global": z["pose_quat_global"][s:s + n], "root_trans_offset": torch.from_numpy(z["root_trans"][s:s + n]),
                             "pose_aa": np.zeros((n, 72)), "fps": 30.0}
        s += n
    return clips


def _hydra_cfg():
    """The tree run_hydra.py builds (EasyDict of cfg.env / cfg.robot / cfg.sim / cfg.learning); plain dicts behave the same."""
    return {"env": {"num_envs": N, "motion_file": _clip_file(20, seed=7), "episode_length": 300, "controlFrequencyInv": 2, "numAMPObsSteps": 10,
                    "local_root_obs": True, "root_height_obs": True, "enableEarlyTermination": True, "terminationDistance": 0.25, "power_reward": True},
            "robot": {"humanoid_type": "smpl", "has_upright_start": True, "has_dof_subset": True},
            "sim": {"dt": 1.0 / 60.0, "substeps": 2, "physx": {"num_threads": 4}},            # the reference's physx block lives under this key
            "seed": 0, "test": False, "im_eval": False, "headless": True}


def test_no_backend_no_silent_fallback():
    backends.register_backend_factory(None)
    with pytest.raises(RuntimeError, match="no simulator backend"):
        HumanoidIm(cfg=_hydra_cfg(), sim_params=None, physics_engine=None, device_type="cuda", device_id=0, headless=True)


def test_parse_task_style_construction_train_epoch_and_resample():
    owners = []
    backends.register_backend_factory(lambda cfg, sim_params, physics_engine, device_type, device_id, headless:
                                      owners.append(FakeGymOwner(cfg["env"]["num_envs"], f"{device_type}:{device_id}")) or owners[-1])
    try:
        cfg = _hydra_cfg()
        sim_params = SimpleNamespace(dt=1.0 / 60.0)
        # parse_task.py:60, keyword for keyword
        task = HumanoidIm(cfg=cfg, sim_params=sim_params, physics_engine="physx", device_type="cuda", device_id=0, headless=True)
        assert task.sim is owners[0] and abs(task.dt - 1.0 / 30.0) < 1e-9 and task.get_obs_size() == 934 and task.get_num_amp_obs() == 1960
        assert task._motion_data.__class__.__name__ == "MotionLibSMPL" and task._motion_lib.num_motions == N      # one clip per env, loaded here
        assert torch.equal(task._pd_action_scale.cpu(), owners[0].pd_action_scale)

        # run_hydra.py:238-240 / create_rlgpu_env: the registries rl_games looks env_name up in
        R.register_vecenv("RLGPU", lambda config_name, num_actors, **kw: SimpleNamespace(
            env=R.configurations[config_name]["env_creator"](**kw), step=None, reset=None))

        class RLGPUEnv:                                          # run_hydra.py:187-236, minus the spaces rl_games reads
            def __init__(self, config_name, num_actors, **kw):
                self.env = R.configurations[config_name]["env_creator"](**kw)

            def step(self, a):
                obs, rew, done, info = self.env.step(a)
                return {"obs": obs}, rew, done, info

            def reset(self, env_ids=None):
                return {"obs": self.env.reset(env_ids)}
        R.register_vecenv("RLGPU", lambda config_name, num_actors, **kw: RLGPUEnv(config_name, num_actors, **kw))
        R.register("rlgpu", {"env_creator": lambda **kw: VecTaskPythonWrapper(task), "vecenv_type": "RLGPU"})

        # what rl_games' Runner hands to the agent factory: params['config'] + the network (here: an object holding the yaml block,
        # like rl_games' model builder does)
        net = SimpleNamespace(network_builder=SimpleNamespace(params={"mlp": {"units": [128, 64], "activation": "relu"},
                                                                      "disc": {"units": [128, 64], "activation": "relu"},
                                                                      "space": {"continuous": {"sigma_init": {"name": "const_initializer", "val": -2.9}}}},
                                                              name="amp"))
        config = {"name": "Humanoid", "env_name": "rlgpu", "env_config": {}, "num_actors": N, "network": net, "horizon_length": 8,
                  "minibatch_size": 128, "amp_minibatch_size": 32, "mini_epochs": 2, "amp_obs_demo_buffer_size": 512, "amp_replay_buffer_size": 512,
                  "amp_batch_size": 64, "learning_rate": 2e-5, "normalize_input": True, "normalize_value": True}

        class IMAmpAgent(AMPAgent):                              # im_amp.py:37-39
            def __init__(self, base_name, config):
                super().__init__(base_name, config)

        agent = IMAmpAgent("run", config)
        assert agent.vec_env.env.task is task and agent.model.actor.layers[0].out_dim == 128 and not agent._graph_rollout
        agent.obs = agent.env_reset()
        agent._init_amp_demo_buf()
        p0 = agent.model.params.clone()
        agent.train_epoch()
        torch.cuda.synchronize()
        assert torch.isfinite(agent.model.params).all() and not torch.equal(agent.model.params, p0) and owners[0].applied > 0
        # the reference's extras['amp_obs'] entry (humanoid_amp.py:207-208) is there for callers that read it
        assert task.extras["amp_obs"].shape == (N, 1960) and torch.equal(task.extras["amp_obs"], task._amp_obs_buf.view(N, -1))

        # resample_motions (humanoid_im.py:369-394): new clips on the device, humanoids stay where they are, every env reset
        torch.manual_seed(5)
        old_keys, old_frames = list(task._motion_data.curr_motion_keys), task._motion_lib.frames_body.clone()
        xy = task._rigid_body_state_reshaped[:, 0, :2].clone()
        task.progress_buf += 3
        task.resample_motions()
        torch.cuda.synchronize()
        assert list(task._motion_data.curr_motion_keys) != old_keys and task._plan.mlib is task._motion_lib
        assert task._motion_lib.frames_body.shape != old_frames.shape or not torch.equal(task._motion_lib.frames_body, old_frames)
        assert int(task.progress_buf.abs().sum()) == 0
        # _global_offset was re-based so that the reference root sits under each humanoid (then reset() re-seats the humanoid on it)
        from phc_b200 import ops
        root = ops.motion_state(task._motion_lib, task._sampled_motion_ids, task._motion_start_times, task._global_offset.contiguous(), want_dof=False)["root_pos"]
        assert torch.allclose(task._rigid_body_state_reshaped[:, 0, :3], root, atol=1e-5)
        agent.obs = agent.env_reset()
        agent.train_epoch()                                       # the plans follow the new tables
        torch.cuda.synchronize()
        assert torch.isfinite(task.obs_buf).all() and torch.isfinite(agent.model.params).all()
    finally:
        backends.register_backend_factory(None)
        R.configurations.pop("rlgpu", None)
        R.vecenv_config.pop("RLGPU", None)


def test_im_amp_eval_sweep_bookkeeping_matches_the_reference_procedure():
    """IMAmpAgent.eval (im_amp.py:136-242) with the bookkeeping on the device (phc_b200/learning/im_amp.py) against the reference's own
    procedure restated literally -- per-step lists of info['mpjpe'] / terminate stacked and sliced per clip on the host
    (_post_step_eval, im_amp.py:244-363) -- fed the same recorded steps: success rate, per-clip MPJPE, failed keys."""
    from phc_b200.learning.im_amp import IMAmpAgent
    n_env, n_clips = 8, 20
    owners = []
    backends.register_backend_factory(lambda cfg, *a: owners.append(FakeGymOwner(cfg["env"]["num_envs"], "cuda:0")) or owners[-1])
    try:
        cfg = _hydra_cfg()
        cfg["env"]["num_envs"] = n_env
        cfg["env"]["motion_file"] = _clip_file(n_clips, seed=11)
        task = HumanoidIm(cfg=cfg, sim_params=SimpleNamespace(dt=1.0 / 60.0), physics_engine="physx", device_type="cuda", device_id=0, headless=True)
        from phc_b200.env.humanoid_im import RLGPUEnv
        agent = IMAmpAgent("run", {"vec_env": RLGPUEnv(task), "horizon_length": 8, "minibatch_size": 64, "amp_minibatch_size": 16, "mini_epochs": 1,
                                   "amp_obs_demo_buffer_size": 256, "amp_replay_buffer_size": 256, "amp_batch_size": 32,
                                   "network": {"mlp": {"units": [64, 32], "activation": "relu"}, "disc": {"units": [64, 32], "activation": "relu"}}})
        agent.obs = agent.env_reset()
        rec = []                                               # what the reference's lists would hold
        real_step = agent.env_eval_step

        def spy(env, actions):
            out = real_step(env, actions)
            lib = task._motion_data
            rec.append(dict(term=out[3]["terminate"].clone().cpu(), mpjpe=out[3]["mpjpe"].clone().cpu(), steps=lib.get_motion_num_steps().cpu(),
                            ids=lib._curr_motion_ids.clone().cpu(), start=task.start_idx))
            return out
        agent.env_eval_step = spy
        info = agent.eval()
        assert set(info) == {"eval/success_rate", "eval/mpjpe_all", "eval/mpjpe_succ"} and task._eval_mode is False
        # --- the reference procedure on the recorded steps
        num_unique = n_clips
        term_mem, mpjpe_all, cur, state, mp = [], [], 0, torch.zeros(n_env, dtype=torch.bool), []
        for r in rec:
            state |= (cur <= r["steps"] - 1) & (r["term"] != 0)
            if (~state).sum() > 0:
                hit = (r["ids"] == num_unique - 1)
                if hit.sum() > 0:
                    bound = int(hit.nonzero()[0]) + 1
                    curr_max = int(r["steps"][:bound][~state[:bound]].max()) if (~state[:bound]).sum() > 0 else cur - 1
                else:
                    curr_max = int(r["steps"][~state].max())
                if cur >= curr_max:
                    curr_max = cur + 1
            else:
                curr_max = int(r["steps"].max())
            mp.append(r["mpjpe"])
            cur += 1
            if cur >= curr_max or int(state.sum()) == n_env:
                cur = 0
                term_mem.append(state.clone())
                allm = torch.stack(mp)
                mpjpe_all.append(torch.stack([allm[:(int(i) - 1), e].mean() for e, i in enumerate(r["steps"])]))
                state, mp = torch.zeros(n_env, dtype=torch.bool), []
        term = torch.cat(term_mem)[:num_unique]
        per_clip = torch.cat(mpjpe_all)[:num_unique]
        assert len(term_mem) == 3                                # 20 clips, 8 at a time
        assert abs(info["eval/success_rate"] - float(1 - term.float().mean())) < 1e-6
        assert abs(info["eval/mpjpe_all"] - float(per_clip.mean()) * 1000) < 1e-2 * max(1.0, float(per_clip.mean()) * 1000) * 1e-2 + 1e-3
        if (~term).any():
            assert abs(info["eval/mpjpe_succ"] - float(per_clip[~term].mean()) * 1000) < 1e-3 + 1e-4 * float(per_clip[~term].mean()) * 1000
    finally:
        backends.register_backend_factory(None)
