"""GPU tests of the rollout's episode statistics and the epoch's learner statistics: phc_episode_stats against the numpy oracle at
rollout sizes, the meters of graph-replayed and eager rollouts, run-to-run repeatability, the per-epoch loss means against the
per-minibatch values of a sequential update, the logit sums of phc_disc_logit_grad, and AMPAgent / IMAmpAgent.train with
`network_path` (checkpoints, tag set, resume, termination history) and without it."""
import os

import numpy as np
import pytest
import torch

from oracle import episode_stats_oracle as EO
from phc_b200 import _lib, ops
from phc_b200 import synthetic as syn
from phc_b200.env.humanoid_im import HumanoidIm, RLGPUEnv
from phc_b200.learning.amp_agent import AMPAgent

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

SMALL = {"horizon_length": 8, "minibatch_size": 256, "amp_minibatch_size": 64, "mini_epochs": 2, "amp_obs_demo_buffer_size": 2048,
         "amp_replay_buffer_size": 2048, "amp_batch_size": 128,
         "network": {"mlp": {"units": [128, 64], "activation": "relu"}, "disc": {"units": [128, 64], "activation": "relu"}}}


def make_agent(n=64, seed=2, cls=AMPAgent, **cfg):
    m = syn.make_motions(n, seed=seed, min_frames=40, max_frames=90)
    task = HumanoidIm({"env": {"num_envs": n}, "motion_data": m, "seed": seed})
    torch.manual_seed(1234)
    return cls("t", dict(SMALL, vec_env=RLGPUEnv(task), **cfg))


# ---- the kernel ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4096, 16384])
def test_kernel_matches_the_oracle_and_the_torch_pair(n):
    rng = np.random.default_rng(n)
    cur_r, cur_l = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    t_r, t_l = cur_r.clone(), cur_l.clone()
    mean, size = torch.zeros(2, device=DEV), torch.zeros(2, dtype=torch.int32, device=DEV)
    gr, gl = EO.AverageMeter(100), EO.AverageMeter(100)
    o_r, o_l = np.zeros(n, np.float32), np.zeros(n, np.float32)
    ks = []
    for p in [0.0, 0.001, 0.01, 0.05, 0.0, 0.2, 0.004, 0.5, 0.0, 0.02, 1.0, 0.003]:
        r = (rng.standard_normal(n) * 0.7 + 0.2).astype(np.float32)
        d = (rng.random(n) < p).astype(np.int64)
        ks.append(int(d.sum()))
        rd, dd = torch.from_numpy(r).to(DEV), torch.from_numpy(d).to(DEV)
        ops.episode_stats(rd, dd, cur_r, cur_l, mean, size, 100)
        not_dones = 1.0 - dd.float()                              # what the rollout ran before the kernel
        t_r.add_(rd).mul_(not_dones)
        t_l.add_(1).mul_(not_dones)
        o_r, o_l = EO.episode_step(o_r, o_l, r, d, gr, gl)
        assert torch.equal(cur_r, t_r) and torch.equal(cur_l, t_l)
        assert torch.equal(cur_r.view(torch.int32), t_r.view(torch.int32))          # signed zeros too
        assert size.tolist() == [gr.current_size, gl.current_size]
        np.testing.assert_allclose(mean.cpu().numpy(), [gr.get_mean(), gl.get_mean()], rtol=2e-6, atol=1e-7)
    assert max(ks) > 100 and 0 < min(k for k in ks if k) < 100 and 0 in ks


def test_kernel_refusals_on_device_tensors():
    n = 64
    args = lambda **kw: {**dict(rewards=torch.zeros(n, device=DEV), dones=torch.zeros(n, dtype=torch.int64, device=DEV),
                                cur_r=torch.zeros(n, device=DEV), cur_l=torch.zeros(n, device=DEV), meter_mean=torch.zeros(2, device=DEV),
                                meter_size=torch.zeros(2, dtype=torch.int32, device=DEV), games_to_track=100), **kw}
    with pytest.raises(TypeError):
        ops.episode_stats(**args(dones=torch.zeros(n, dtype=torch.int32, device=DEV)))
    with pytest.raises(TypeError):
        ops.episode_stats(**args(meter_size=torch.zeros(2, device=DEV)))
    with pytest.raises(ValueError, match="contiguous"):
        ops.episode_stats(**args(rewards=torch.zeros(n, 2, device=DEV)[:, 0]))
    with pytest.raises(_lib.PhcError, match="games_to_track"):
        ops.episode_stats(**args(games_to_track=0))


# ---- the agent: meters ------------------------------------------------------------------------------------------------------
def test_graph_replayed_and_eager_rollouts_leave_identical_meters():
    agents = []
    for graphed in (False, True):
        ag = make_agent(graph_rollout=graphed, games_to_track=20)
        ag.obs = ag.env_reset()
        ag._init_amp_demo_buf()
        agents.append(ag)
    assert agents[1]._graph_rollout and not agents[0]._graph_rollout
    for epoch in range(8):
        for ag in agents:
            torch.manual_seed(77 + epoch)
            ag.set_eval()
            ag.play_steps()
        torch.cuda.synchronize()
        for k in ("_meter_mean", "_meter_size", "current_rewards", "current_lengths"):
            assert torch.equal(getattr(agents[0], k), getattr(agents[1], k)), f"epoch {epoch}: {k}"
    assert agents[1]._rollout_graph is not None
    assert agents[0].game_rewards.current_size > 0, "no episode finished in 64 steps: the comparison saw empty meters"


def test_two_runs_give_bit_identical_meters_and_epoch_statistics():
    out = []
    for _ in range(2):
        ag = make_agent()
        ag.obs = ag.env_reset()
        ag._init_amp_demo_buf()
        infos = [ag.train_epoch() for _ in range(3)]
        torch.cuda.synchronize()
        out.append((ag._meter_mean.clone(), ag._meter_size.clone(), [i["epoch_stats"]["loss_means"] for i in infos], ag._epoch_stats.clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    assert all(torch.equal(a, b) for a, b in zip(out[0][2], out[1][2]))
    assert torch.equal(out[0][3], out[1][3])


def test_epoch_loss_means_equal_the_mean_of_per_minibatch_values(monkeypatch):
    """One agent updates through the pipeline; its twin runs the same minibatches one calc_gradients at a time and reads
    train_result_dict() after each.  Same stream, same order: the same per-minibatch statistics, and the epoch means are their
    means."""
    pipelined, sequential = make_agent(), make_agent()
    collected = []

    def one_at_a_time():
        mb = sequential.minibatch_size
        for _ in range(sequential.mini_epochs_num):
            for i in range(sequential.num_minibatches):
                sequential.calc_gradients({"idx": sequential._idx_buf[i * mb:(i + 1) * mb]})
                s, Bd = sequential._stats.tolist(), sequential._amp_minibatch_size
                collected.append(dict(sequential.train_result_dict(), disc_agent_logit=s[13] / (2 * Bd), disc_demo_logit=s[14] / Bd))
            sequential._idx_buf = torch.randperm(sequential.batch_size, device=sequential.device)
    monkeypatch.setattr(sequential, "_minibatch_pipeline", one_at_a_time)
    for ag in (pipelined, sequential):
        torch.manual_seed(5)
        ag.obs = ag.env_reset()
        ag._init_amp_demo_buf()
        ag.train_epoch()
    collected.clear()
    torch.manual_seed(6)
    sequential.train_epoch()
    torch.manual_seed(6)
    info_p = pipelined.train_epoch()
    torch.cuda.synchronize()
    M = pipelined.mini_epochs_num * pipelined.num_minibatches
    assert len(collected) == M == pipelined._epoch_stats.shape[0] and M > 1
    means = dict(zip(AMPAgent._STAT_KEYS, info_p["epoch_stats"]["loss_means"].tolist()))
    for k in collected[0]:
        exp = float(np.mean([c[k] for c in collected]))
        assert means[k] == pytest.approx(exp, rel=1e-6, abs=1e-9), k
    last = {k: v for k, v in collected[-1].items() if k not in ("disc_agent_logit", "disc_demo_logit")}
    assert pipelined.train_result_dict() == last                           # train_result_dict: still the last minibatch, same keys


def test_disc_logit_sums_against_torch_and_the_other_slots_unchanged():
    g = torch.Generator(device=DEV).manual_seed(9)
    na, nd = 8192, 4096
    logit = torch.randn(na + nd, device=DEV, generator=g) * 2
    dl = torch.zeros(na + nd, device=DEV)
    stats = torch.zeros(16, device=DEV)
    _lib.check(_lib.load().phc_disc_logit_grad(logit.data_ptr(), 1, na, nd, 5.0, dl.data_ptr(), 1, stats.data_ptr(), None))
    s = stats.double().cpu()
    x = logit.double().cpu()
    assert s[13].item() == pytest.approx(float(x[:na].sum()), rel=1e-5, abs=1e-2)
    assert s[14].item() == pytest.approx(float(x[na:].sum()), rel=1e-5, abs=1e-2)
    sp = torch.nn.functional.softplus(x)
    assert s[6].item() == pytest.approx(float(sp[:na].sum()), rel=1e-5) and s[7].item() == pytest.approx(float((sp[na:] - x[na:]).sum()), rel=1e-5)
    assert s[8] == float((x[:na] < 0).sum()) and s[9] == float((x[na:] > 0).sum())
    assert s[10:13].abs().sum() == 0 and s[15] == 0 and s[:6].abs().sum() == 0


# ---- the agent: the training loop ----------------------------------------------------------------------------------------
class Recorder:
    def __init__(self):
        self.calls = []

    def add_scalar(self, tag, value, step):
        self.calls.append((tag, float(value), step))


TAGS = {"performance/total_fps", "performance/step_fps", "performance/update_time", "performance/play_time", "episode_lengths/epochs",
        "episode_lengths/frame", "episode_lengths/iter", "rewards0/frame", "rewards0/iter", "rewards0/time", "rewards/mean_rewards",
        "loss/actor_loss", "loss/critic_loss", "loss/bounds_loss", "loss/entropy", "loss/clip_frac", "loss/kl", "disc/loss",
        "disc/agent_acc", "disc/demo_acc", "disc/agent_logit", "disc/demo_logit", "disc/grad_penalty", "disc/logit_loss",
        "disc/reward_mean", "disc/reward_std", "rewards/returns", "rewards/mb_rewards", "rewards/body_pos", "rewards/body_rot",
        "rewards/lin_vel", "rewards/ang_vel", "rewards/power", "learning_rate/last_lr", "learning_rate/lr_mul", "learning_rate/e_clip"}


def test_train_with_network_path_saves_logs_and_resumes(tmp_path, monkeypatch):
    import joblib
    from phc_b200.learning.im_amp import IMAmpAgent
    rec = Recorder()
    ag = make_agent(cls=IMAmpAgent, network_path=str(tmp_path), save_best_after=2, save_frequency=3, save_intermediate=True,
                    max_epochs=4, writer=rec)
    evals = []
    monkeypatch.setattr(ag, "eval", lambda: (evals.append(ag.epoch_num), {"eval/success_rate": 0.5})[1])
    ag._meter_size.fill_(1)                    # as if an episode had ended before the run: every epoch logs the reward scalars
    ag.train()
    assert ag.epoch_num == 5
    assert sorted(os.listdir(tmp_path)) == ["Humanoid.pth", "Humanoid_00000003.pth"]
    assert evals == [3]
    tags = {t for t, _, _ in rec.calls}
    assert TAGS <= tags and "eval/success_rate" in tags
    vals = {(t, s): v for t, v, s in rec.calls}
    assert all(np.isfinite(v) for v in vals.values())
    assert 0.0 <= vals[("disc/agent_acc", 5)] <= 1.0 and vals[("learning_rate/lr_mul", 5)] == 1.0
    ck = torch.load(tmp_path / "Humanoid.pth", map_location=DEV, weights_only=False)
    assert ck["epoch"] == 5                     # the final save

    # resume: a new agent restores the checkpoint and continues the epoch count; the newest failed_*.pkl sets the sampling weights
    hist = torch.arange(1, 9, dtype=torch.float32, device=DEV)
    joblib.dump({"failed_keys": [], "termination_history": hist * 0 + 1}, tmp_path / "failed_0000000003.pkl")
    joblib.dump({"failed_keys": [], "termination_history": hist}, tmp_path / "failed_0000000012.pkl")
    rec2 = Recorder()
    ag2 = make_agent(cls=IMAmpAgent, network_path=str(tmp_path), save_best_after=2, save_frequency=3, max_epochs=6, writer=rec2)
    got = []
    monkeypatch.setattr(type(ag2.vec_env.env.task._motion_data), "update_sampling_prob",
                        lambda self, th: (got.append(th.clone()), True)[1], raising=False)
    ag2.restore(str(tmp_path / "Humanoid.pth"))
    ag2._meter_size.fill_(1)
    assert ag2.epoch_num == 5 and len(got) == 1 and torch.equal(got[0], hist)
    assert torch.equal(ag2.model.params, ag.model.params)
    ag2.train()
    assert ag2.epoch_num == 7 and {s for t, _, s in rec2.calls if t == "loss/kl"} == {6, 7}


def test_train_without_network_path_writes_nothing(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    ag = make_agent(save_best_after=1, save_frequency=1, save_intermediate=True)
    info = ag.train(max_epochs=2)
    torch.cuda.synchronize()
    assert ag.epoch_num == 2 and list(tmp_path.iterdir()) == []
    assert {"play_time", "update_time", "total_time", "returns", "disc_rewards", "epoch_stats"} <= set(info)
    # the tensors train_epoch hands back at the top level are the ones it returned before the epoch statistics existed
    assert {k for k, v in info.items() if torch.is_tensor(v)} == {"terminated_flags", "reward_raw", "mb_rewards", "returns", "disc_rewards"}
