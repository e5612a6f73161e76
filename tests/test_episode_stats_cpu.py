"""The rollout's episode statistics without a GPU: rl_games' AverageMeter rule as restated by oracle/episode_stats_oracle.py on
hand-computed cases (no dones, one done, more dones than games_to_track, the meter filling up over several steps), then the kernel
source of phc_b200/csrc/episode_stats.cu through the CPU emulation of tests/emu against that oracle over a random multi-step done
pattern (one run with every lane dawdling after each collective), and the refusals of the wrapper and of the C ABI."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

from oracle import episode_stats_oracle as EO                       # noqa: E402


def _meters(max_size):
    return EO.AverageMeter(max_size), EO.AverageMeter(max_size)


# ---- the oracle on hand-computed cases ------------------------------------------------------------------------------------
def test_no_dones_leaves_the_meters_alone():
    gr, gl = _meters(100)
    cr, cl = EO.episode_step(np.array([1.0, 2.0], np.float32), np.array([3.0, 4.0], np.float32), np.array([0.5, -1.0], np.float32),
                             np.array([0, 0]), gr, gl)
    assert cr.tolist() == [1.5, 1.0] and cl.tolist() == [4.0, 5.0]
    assert gr.current_size == 0 and gl.current_size == 0 and gr.get_mean() == 0.0 and gl.get_mean() == 0.0


def test_one_done():
    gr, gl = _meters(100)
    cr, cl = EO.episode_step(np.array([1.0, 2.0, 3.0], np.float32), np.array([4.0, 5.0, 6.0], np.float32),
                             np.array([0.5, 0.5, 0.5], np.float32), np.array([0, 1, 0]), gr, gl)
    assert cr.tolist() == [1.5, 0.0, 3.5] and cl.tolist() == [5.0, 0.0, 7.0]
    assert (gr.current_size, gr.get_mean()) == (1, 2.5) and (gl.current_size, gl.get_mean()) == (1, 6.0)


def test_more_dones_than_games_to_track_take_the_mean_of_all():
    """max_size 2, the meter full at mean 10, three episodes end with returns 1, 2, 6: old = 0 and the meter becomes their mean
    3 (not 1.5, the mean of the first two)."""
    gr, gl = _meters(2)
    gr.update([10.0, 10.0])
    gl.update([8.0, 8.0])
    assert gr.current_size == 2 and gr.get_mean() == 10.0
    cr, _ = EO.episode_step(np.array([1.0, 2.0, 6.0, 9.0], np.float32), np.zeros(4, np.float32), np.zeros(4, np.float32),
                            np.array([1, 1, 1, 0]), gr, gl)
    assert (gr.current_size, gr.get_mean()) == (2, 3.0) and (gl.current_size, gl.get_mean()) == (2, 1.0)
    assert cr.tolist() == [0.0, 0.0, 0.0, 9.0]


def test_meter_fills_up_over_several_steps():
    """max_size 3: values 4 | 7 | 1, 3 | 10 over four steps."""
    g = EO.AverageMeter(3)
    g.update([4.0])
    assert (g.current_size, g.get_mean()) == (1, 4.0)
    g.update([7.0])                                           # old = min(2, 1) = 1: (4 + 7) / 2
    assert (g.current_size, g.get_mean()) == (2, 5.5)
    g.update([1.0, 3.0])                                      # size 2, old = min(1, 2) = 1: (5.5 + 2 * 2) / 3
    assert g.current_size == 3 and g.get_mean() == pytest.approx(9.5 / 3, rel=1e-6)
    g.update([10.0])                                          # size 1, old = min(2, 3) = 2: (2 * 9.5 / 3 + 10) / 3
    assert g.current_size == 3 and g.get_mean() == pytest.approx((2 * 9.5 / 3 + 10.0) / 3, rel=1e-6)
    g.update([])
    assert g.current_size == 3


# ---- the kernel source under the CPU emulation ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    import shutil
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    import episode_stats_emu
    return episode_stats_emu.EmuEpisodeStats(episode_stats_emu.build(str(tmp_path_factory.mktemp("emu_episode_stats"))))


def done_pattern(rng, n, steps):
    """per step a different done rate: none, a few, and more than 100 of n"""
    rates = [0.0, 0.002, 0.05, 0.3, 0.0, 0.01, 0.5, 0.001, 0.2, 0.0, 0.08, 1.0][:steps]
    return [(rng.random(n) < p).astype(np.int64) for p in rates]


@pytest.mark.parametrize("n,games", [(1500, 100), (37, 5), (600, 1)])
def test_emulated_kernel_matches_the_oracle(emu, n, games):
    rng = np.random.default_rng(n + games)
    cur_r, cur_l = torch.zeros(n), torch.zeros(n)
    mean, size = torch.zeros(2), torch.zeros(2, dtype=torch.int32)
    gr, gl = _meters(games)
    o_r, o_l = np.zeros(n, np.float32), np.zeros(n, np.float32)
    for d in done_pattern(rng, n, 12):
        r = (rng.standard_normal(n) * 0.7 + 0.2).astype(np.float32)
        emu.step(torch.from_numpy(r), torch.from_numpy(d), cur_r, cur_l, mean, size, games)
        o_r, o_l = EO.episode_step(o_r, o_l, r, d, gr, gl)
        assert np.array_equal(cur_r.numpy().view(np.int32), o_r.view(np.int32))        # bit for bit, signed zeros included
        assert np.array_equal(cur_l.numpy(), o_l)
        assert size.tolist() == [gr.current_size, gl.current_size]
        np.testing.assert_allclose(mean.numpy(), [gr.get_mean(), gl.get_mean()], rtol=2e-6, atol=1e-7)
    assert gr.current_size == min(games, n)


def test_emulated_kernel_repeats_bit_for_bit(emu):
    rng = np.random.default_rng(5)
    n = 2000
    r, d = torch.from_numpy(rng.standard_normal(n).astype(np.float32)), torch.from_numpy((rng.random(n) < 0.4).astype(np.int64))
    out = []
    for _ in range(2):
        cur_r, cur_l = torch.full((n,), 0.25), torch.full((n,), 3.0)
        mean, size = torch.tensor([1.5, 7.0]), torch.tensor([40, 40], dtype=torch.int32)
        emu.step(r, d, cur_r, cur_l, mean, size, 100)
        out.append(torch.cat((cur_r, cur_l, mean)))
    assert torch.equal(out[0], out[1])


def test_episode_stats_chaos_mode_subset():
    """The same emulation with every lane dawdling randomly after each collective (PHC_EMU_CHAOS=1, read when the emulation library
    loads, hence a fresh process)."""
    import subprocess
    if os.environ.get("PHC_EMU_CHAOS") == "1":
        pytest.skip("already inside the chaos run")
    env = dict(os.environ, PHC_EMU_CHAOS="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-p", "no:cacheprovider", "-k",
                        "emulated_kernel_matches and 1500"], capture_output=True, text=True, env=env, cwd=os.path.dirname(HERE), timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


# ---- refusals -----------------------------------------------------------------------------------------------------------
def test_wrapper_refuses_cpu_tensors():
    from phc_b200 import ops
    n = 4
    with pytest.raises(ops.PhcError):
        ops.episode_stats(torch.zeros(n), torch.zeros(n, dtype=torch.int64), torch.zeros(n), torch.zeros(n), torch.zeros(2),
                          torch.zeros(2, dtype=torch.int32), 100)


def test_c_abi_refuses_bad_input():
    """phc_episode_stats validates before it launches: n <= 0, games_to_track < 1, NULL pointers."""
    from phc_b200 import _lib
    lib = _lib.load()
    p = 256                                              # never dereferenced: every call below is refused first
    for n, games, ptrs in ((0, 100, [p] * 6), (-2, 100, [p] * 6), (4, 0, [p] * 6), (4, -1, [p] * 6), (4, 100, [p, None, p, p, p, p]),
                           (4, 100, [p, p, p, p, p, None])):
        assert lib.phc_episode_stats(ptrs[0], ptrs[1], n, ptrs[2], ptrs[3], ptrs[4], ptrs[5], games, None) == -1, (n, games, ptrs)
        assert lib.phc_last_error().decode().startswith("phc_episode_stats")
