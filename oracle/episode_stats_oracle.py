"""numpy restatement of the rollout's episode bookkeeping: AMPAgent.play_steps (phc/learning/amp_agent.py:358-369) with rl_games
1.1.4's `AverageMeter` (rl_games/algos_torch/torch_ext.py).  rl_games is neither in the reference tree nor installable here, so the
meter rule is written from the published class and pinned by hand-computed cases (tests/test_episode_stats_cpu.py):

    def update(self, values):
        size = values.size()[0]
        if size == 0: return
        new_mean = torch.mean(values.float(), dim=0)
        size = np.clip(size, 0, self.max_size)
        old_size = min(self.max_size - size, self.current_size)
        size_sum = old_size + size
        self.current_size = size_sum
        self.mean = (self.mean * old_size + new_mean * size) / size_sum

The new mean is over ALL done values, not the first max_size of them; when a step ends max_size episodes or more, old_size is 0 and
the meter becomes the mean of that step alone.  The meter keeps fp32 (its `mean` buffer); the batch mean is taken here in fp64.
"""
from __future__ import annotations

import numpy as np


class AverageMeter:
    def __init__(self, max_size: int):
        assert max_size >= 1
        self.max_size = int(max_size)
        self.current_size = 0
        self.mean = np.float32(0.0)

    def update(self, values) -> None:
        values = np.asarray(values, dtype=np.float64).reshape(-1)
        k = values.shape[0]
        if k == 0:
            return
        new_mean = np.float32(values.mean())
        size = min(k, self.max_size)
        old = min(self.max_size - size, self.current_size)
        self.current_size = old + size
        self.mean = np.float32((np.float32(self.mean * np.float32(old)) + np.float32(new_mean * np.float32(size))) / np.float32(old + size))

    def get_mean(self) -> float:
        return float(self.mean)


def episode_step(cur_r: np.ndarray, cur_l: np.ndarray, rewards: np.ndarray, dones: np.ndarray, game_rewards: AverageMeter,
                 game_lengths: AverageMeter):
    """One rollout step: returns the new (cur_r, cur_l) fp32 arrays and updates the two meters in place."""
    v_r = (cur_r.astype(np.float32) + rewards.astype(np.float32)).astype(np.float32)
    v_l = (cur_l.astype(np.float32) + np.float32(1.0)).astype(np.float32)
    done = np.asarray(dones) != 0
    game_rewards.update(v_r[done])
    game_lengths.update(v_l[done])
    not_done = (np.float32(1.0) - np.asarray(dones).astype(np.float32)).astype(np.float32)
    return (v_r * not_done).astype(np.float32), (v_l * not_done).astype(np.float32)
