"""AMPAgent.train's checkpoint / evaluation / logging cadence (CommonAgent.train, common_agent.py:100-185) without a GPU: the loop runs
on a stub agent whose epochs only advance the counters and whose device read-back is replaced by fixed host values, so what is
checked is which epochs save, evaluate and log, the tag set, and that nothing of it runs without `network_path`."""
import pytest

from phc_b200.learning.amp_agent import AMPAgent


class Recorder:
    def __init__(self):
        self.calls = []

    def add_scalar(self, tag, value, step):
        self.calls.append((tag, value, step))

    def tags_at(self, step):
        return {t for t, _, s in self.calls if s == step}


def stub_agent(monkeypatch, cfg, game_size_from=1, rank=0):
    ag = AMPAgent.__new__(AMPAgent)
    ag.config = {**dict(name="Humanoid", max_epochs=10000000, save_frequency=2500, save_best_after=100), **cfg}
    ag.rank, ag.world, ag.batch_size, ag.frame, ag.epoch_num = rank, 1, 256, 0, 0
    ag.e_clip, ag.last_lr = 0.2, 2e-5
    ag._disc_logit_reg, ag._disc_grad_penalty, ag._disc_weight_decay = 0.01, 5.0, 1e-4
    ag.saved, ag.evaluated = [], []
    monkeypatch.setattr(ag, "env_reset", lambda *a: {}, raising=False)
    monkeypatch.setattr(ag, "_init_amp_demo_buf", lambda: None, raising=False)

    def train_epoch():
        ag.epoch_num += 1
        ag.frame += ag.batch_size
        return dict(play_time=0.5, update_time=0.25, total_time=0.75, last_lr=ag.last_lr, lr_mul=1.0)

    def read(info):
        host = {k: 0.5 for k in AMPAgent._STAT_KEYS}
        host.update(game_rewards=12.0, game_lengths=30.0, game_size=5 if ag.epoch_num >= game_size_from else 0, returns=1.0,
                    mb_rewards=0.1, disc_reward_std=0.2, disc_reward_mean=0.3, reward_raw=[0.1, 0.2, 0.3, 0.4, 0.5])
        info["host"] = host
        return host

    monkeypatch.setattr(ag, "train_epoch", train_epoch, raising=False)
    monkeypatch.setattr(ag, "_read_epoch_scalars", read, raising=False)
    monkeypatch.setattr(ag, "save", lambda fn: ag.saved.append((ag.epoch_num, fn)), raising=False)
    monkeypatch.setattr(ag, "eval", lambda: (ag.evaluated.append(ag.epoch_num), {"eval/success_rate": 0.75})[1], raising=False)
    return ag


REFERENCE_TAGS = {
    "performance/total_fps", "performance/step_fps", "performance/update_time", "performance/play_time", "episode_lengths/epochs",
    "episode_lengths/frame", "episode_lengths/iter", "episode_lengths/episode_lengths", "rewards0/frame", "rewards0/iter",
    "rewards0/time", "rewards/mean_rewards", "loss/actor_loss", "loss/critic_loss", "loss/bounds_loss", "loss/entropy",
    "loss/clip_frac", "loss/kl", "disc/loss", "disc/agent_acc", "disc/demo_acc", "disc/agent_logit", "disc/demo_logit",
    "disc/grad_penalty", "disc/logit_loss", "disc/reward_mean", "disc/reward_std", "rewards/returns", "rewards/mb_rewards",
    "rewards/body_pos", "rewards/body_rot", "rewards/lin_vel", "rewards/ang_vel", "rewards/power", "learning_rate/last_lr",
    "learning_rate/lr_mul", "learning_rate/e_clip"}


def test_save_eval_and_log_epochs(monkeypatch, tmp_path):
    """save_best_after 3, save_frequency 4, save_intermediate, max_epochs 9; episodes have finished from epoch 5 on:
    <name>.pth at 3, 6, 9 and the final save at 10; <name>_<epoch:08d>.pth at 4 and 8; eval only at 8 (no finished episode at 4);
    reward / length / loss scalars from epoch 5 on; the performance scalars every epoch."""
    rec = Recorder()
    ag = stub_agent(monkeypatch, dict(network_path=str(tmp_path), save_best_after=3, save_frequency=4, save_intermediate=True,
                                      max_epochs=9, writer=rec), game_size_from=5)
    ag.train()
    base = str(tmp_path / "Humanoid")
    assert ag.saved == [(3, base), (4, base + "_00000004"), (6, base), (8, base + "_00000008"), (9, base), (10, base)]
    assert ag.epoch_num == 10 and ag.evaluated == [8]
    for e in range(1, 11):
        # add_scalar steps: the frame for performance/*, episode_lengths/epochs, rewards0/frame, episode_lengths/frame; else the epoch
        frame_tags = {t for t, _, s in rec.calls if s == (e - 1) * 256 and t in ("performance/total_fps", "performance/step_fps",
                                                                                  "episode_lengths/epochs")}
        assert len(frame_tags) == 3 or e == 1
        logged = rec.tags_at(e)
        if e < 5:
            assert not any(t.startswith(("loss/", "disc/", "rewards")) for t in logged), e
        else:
            assert REFERENCE_TAGS - {"performance/total_fps", "performance/step_fps", "episode_lengths/epochs", "rewards0/frame",
                                     "episode_lengths/frame", "rewards0/time"} <= logged, e
            assert ("eval/success_rate" in logged) == (e == 8)
    every = {t for t, _, _ in rec.calls}
    assert REFERENCE_TAGS <= every
    assert ("episode_lengths/epochs", 10, 9 * 256) in rec.calls
    assert ("rewards0/iter", 12.0, 7) in rec.calls and ("episode_lengths/iter", 30.0, 7) in rec.calls
    # disc/loss: the reference's total (BCE + logit regulariser + gradient penalty + weight decay) from the minibatch means
    assert ("disc/loss", 0.5 + 0.01 * 0.5 + 5.0 * 0.5 + 1e-4 * 0.5, 7) in rec.calls


def test_without_save_intermediate_only_the_latest_checkpoint(monkeypatch, tmp_path):
    rec = Recorder()
    ag = stub_agent(monkeypatch, dict(network_path=str(tmp_path), save_best_after=100, save_frequency=2, max_epochs=4, writer=rec))
    ag.train()
    assert [e for e, _ in ag.saved] == [5] and ag.evaluated == []          # min(50, 100) = 50: only the final save


def test_other_ranks_neither_save_nor_log(monkeypatch, tmp_path):
    rec = Recorder()
    ag = stub_agent(monkeypatch, dict(network_path=str(tmp_path), save_best_after=1, save_frequency=1, save_intermediate=True,
                                      max_epochs=3, writer=rec), rank=1)
    ag.train()
    assert ag.epoch_num == 4 and ag.saved == [] and ag.evaluated == [] and rec.calls == []


def test_without_network_path_nothing_is_written(monkeypatch, tmp_path):
    rec = Recorder()
    monkeypatch.chdir(tmp_path)
    ag = stub_agent(monkeypatch, dict(save_best_after=1, save_frequency=1, save_intermediate=True, writer=rec))
    ag.train(max_epochs=3)
    assert ag.epoch_num == 3 and ag.saved == [] and ag.evaluated == [] and rec.calls == []
    assert list(tmp_path.iterdir()) == []


def test_console_line(monkeypatch, tmp_path, capsys):
    ag = stub_agent(monkeypatch, dict(network_path=str(tmp_path), train_dir=str(tmp_path / "run7"), max_epochs=1, writer=Recorder()))
    ag.train()
    out = capsys.readouterr().out
    assert "run7-Ep: 1\trwd: 12.0\t" in out and "eps_len: 30.0" in out and "MAX EPOCHS NUM!" in out
