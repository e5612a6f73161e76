"""The imitation evaluation metrics on the GPU: phc_eval_metrics_step through the C ABI against the fp64 oracle
(oracle/eval_metrics_oracle.py) on the cases of the CPU emulation test plus 4096 envs, bit-identical from run to run; and
IMAmpAgent.eval(full_eval_metrics=True) on the fake simulator owner of test_gpu_dropin_construct.py against the reference's own
procedure restated literally on the host (per-step lists of body_pos / body_pos_gt stacked, sliced [:num_steps - 1] per clip,
concatenated, cut to the unique clips, then compute_metrics_lite)."""
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import eval_metrics_oracle as EO
from phc_b200 import ops
from tests import eval_metrics_cases as EC

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEYS8 = {"eval/success_rate", "eval/mpjpe_all", "eval/mpjpe_succ", "eval/accel_dist", "eval/vel_dist", "eval/mpjpel_all",
         "eval/mpjpel_succ", "eval/mpjpe_pa"}


def _to(dev, *ts):
    return [t.to(dev) for t in ts]


@pytest.mark.parametrize("case", EC.CASES, ids=[c[0] for c in EC.CASES])
def test_kernel_matches_the_oracle(case):
    _, n, J, B, S = case
    state, gt, ns = EC.make_case(n, J, B, S, seed=J + B)
    acc, _ = EC.run(ops.eval_metrics_step, *_to(DEV, state, gt, ns), J)
    EC.compare(acc, EC.expected(state, gt, ns, J))


@pytest.mark.parametrize("J", [20, 52])
def test_kernel_undoes_a_known_similarity(J):
    state, gt, ns = EC.make_case(5, J, J, 5, seed=J, num_steps=[9] * 5, kind="similar")
    acc, _ = EC.run(ops.eval_metrics_step, *_to(DEV, state, gt, ns), J)
    got = acc.cpu().numpy()
    assert np.all(got[:, 5] == 5) and np.all(got[:, 2] / got[:, 5] < 2e-6) and np.all(got[:, 0] / got[:, 5] > 1e-2)
    EC.compare(acc, EC.expected(state, gt, ns, J))


def test_kernel_40_steps_two_batches():
    n, J = 6, 24
    state, gt, ns = EC.make_case(n, J, J, 40, seed=40, num_steps=[1, 2, 3, 20, 26, 40])
    s, g, nd = _to(DEV, state, gt, ns)
    acc, ring = EC.run(ops.eval_metrics_step, s[:25], g[:25], nd, J)
    EC.compare(acc, EC.expected(state[:25], gt[:25], ns, J))
    acc2, _ = EC.run(ops.eval_metrics_step, s[25:], g[25:], nd, J, ring=ring)
    EC.compare(acc2, EC.expected(state[25:], gt[25:], ns, J))


def test_kernel_4096_envs_bit_identical_across_runs():
    n, J, S = 4096, 24, 6
    state, gt, ns = EC.make_case(n, J, J, S, seed=4096)
    s, g, nd = _to(DEV, state, gt, ns)
    acc1, ring1 = EC.run(ops.eval_metrics_step, s, g, nd, J)
    acc2, ring2 = EC.run(ops.eval_metrics_step, s, g, nd, J)
    torch.cuda.synchronize()
    assert torch.equal(acc1, acc2) and torch.equal(ring1, ring2)
    EC.compare(acc1, EC.expected(state, gt, ns, J))


def test_c_abi_refusals_on_device_tensors():
    n, J = 4, 24
    pos = torch.zeros(n, 70, 3, device=DEV)
    args = (torch.zeros(n, 70, 3, device=DEV), torch.ones(n, dtype=torch.int32, device=DEV), 0, torch.zeros(2, n, 70, 3, device=DEV),
            torch.zeros(n, 8, dtype=torch.float64, device=DEV))
    with pytest.raises(ValueError):
        ops.eval_metrics_step(pos, *args)
    with pytest.raises(ValueError):                       # x, y, z not contiguous
        ops.eval_metrics_step(torch.zeros(n, 3, J, device=DEV).transpose(1, 2), torch.zeros(n, J, 3, device=DEV), args[1], 0,
                              torch.zeros(2, n, J, 3, device=DEV), args[4])


# ---- IMAmpAgent.eval -------------------------------------------------------------------------------------------------------
def _tracking_owner_cls():
    from tests.test_gpu_dropin_construct import FakeGymOwner, J

    class TrackingOwner(FakeGymOwner):
        """simulate() puts every body at the reference pose the next env step compares against, plus a fixed noise pattern (a
        function of the step and the clip, so two sweeps see the same inputs); clips with motion id % 3 == 1 are pushed 1 m away
        from the reference after their fifth step and fail."""
        task = None

        def simulate(self, actions):
            super().simulate(actions)
            task = self.task
            if task is None or not getattr(task, "_eval_mode", False):
                return
            if not hasattr(self, "_noise"):
                g = torch.Generator().manual_seed(9)
                self._noise = (torch.randn(128, 64, J, 3, generator=g) * 0.02).to(self.rigid_body_state.device)
            prog = task.progress_buf + 1
            ids = task._sampled_motion_ids
            t = prog.float() * task.dt + task._motion_start_times + task._motion_start_times_offset
            pos = ops.motion_state(task._motion_lib, ids, t.contiguous(), task._global_offset.contiguous(), want_dof=False)["rg_pos"]
            pos = pos + self._noise[prog % 128, ids % 64]
            push = ((ids % 3) == 1) & (prog > 5)
            pos[..., 2] += torch.where(push, 1.0, 0.0)[:, None]
            self.rigid_body_state[:, :J, 0:3] = pos
    return TrackingOwner


def _make_agent(full, n_env=8, n_clips=20):
    from phc_b200.env import backends
    from phc_b200.env.humanoid_im import HumanoidIm, RLGPUEnv
    from phc_b200.learning.im_amp import IMAmpAgent
    from tests.test_gpu_dropin_construct import _clip_file, _hydra_cfg
    Owner = _tracking_owner_cls()
    owners = []
    torch.manual_seed(0)
    np.random.seed(0)                                     # MotionLibSMPL.load_motions draws a random heading per clip
    random.seed(0)
    backends.register_backend_factory(lambda cfg, *a: owners.append(Owner(cfg["env"]["num_envs"], DEV)) or owners[-1])
    try:
        cfg = _hydra_cfg()
        cfg["env"]["num_envs"] = n_env
        cfg["env"]["motion_file"] = _clip_file(n_clips, seed=11)
        task = HumanoidIm(cfg=cfg, sim_params=SimpleNamespace(dt=1.0 / 60.0), physics_engine="physx", device_type="cuda", device_id=0, headless=True)
    finally:
        backends.register_backend_factory(None)
    owners[0].task = task
    torch.manual_seed(0)
    agent = IMAmpAgent("run", {"vec_env": RLGPUEnv(task), "horizon_length": 8, "minibatch_size": 64, "amp_minibatch_size": 16, "mini_epochs": 1,
                               "amp_obs_demo_buffer_size": 256, "amp_replay_buffer_size": 256, "amp_batch_size": 32, "full_eval_metrics": full,
                               "network": {"mlp": {"units": [64, 32], "activation": "relu"}, "disc": {"units": [64, 32], "activation": "relu"}}})
    agent.obs = agent.env_reset()
    return agent, task


def _spy_eval(agent, task):
    """agent.eval() with every step's extras recorded on the host (what the reference's lists would hold), and the failed keys."""
    rec, failed = [], []
    real_step, real_update = agent.env_eval_step, agent.update_training_data

    def spy(env, actions):
        out = real_step(env, actions)
        lib = task._motion_data
        rec.append(dict(term=out[3]["terminate"].clone().cpu(), mpjpe=out[3]["mpjpe"].clone().cpu(), steps=lib.get_motion_num_steps().cpu(),
                        ids=lib._curr_motion_ids.clone().cpu(), pred=out[3]["body_pos"].clone().cpu(), gt=out[3]["body_pos_gt"].clone().cpu()))
        return out
    agent.env_eval_step = spy
    agent.update_training_data = lambda keys: failed.append(list(keys)) or real_update(keys)
    try:
        info = agent.eval()
    finally:
        agent.env_eval_step, agent.update_training_data = real_step, real_update
    return info, rec, failed[0]


def _reference_procedure(rec, n_env, num_unique):
    """_post_step_eval (im_amp.py:244-363) on the recorded steps: the batch bookkeeping of the existing test, plus the stacked body
    positions sliced per clip; returns (terminated [num_unique], per-clip MPJPE [num_unique], pred clips, gt clips)."""
    term_mem, mpjpe_all, pred_all, gt_all = [], [], [], []
    cur, state, mp, pp, gp = 0, torch.zeros(n_env, dtype=torch.bool), [], [], []
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
        pp.append(r["pred"].numpy())
        gp.append(r["gt"].numpy())
        cur += 1
        if cur >= curr_max or int(state.sum()) == n_env:
            cur = 0
            term_mem.append(state.clone())
            allm = torch.stack(mp)
            mpjpe_all.append(torch.stack([allm[:(int(i) - 1), e].mean() for e, i in enumerate(r["steps"])]))
            p_clips, g_clips = EO.slice_batch(np.stack(pp), np.stack(gp), r["steps"].tolist())
            pred_all += p_clips
            gt_all += g_clips
            state, mp, pp, gp = torch.zeros(n_env, dtype=torch.bool), [], [], []
    term = torch.cat(term_mem)[:num_unique].numpy()
    return term, torch.cat(mpjpe_all)[:num_unique], pred_all[:num_unique], gt_all[:num_unique], len(term_mem)


def test_im_amp_full_eval_metrics_match_the_reference_procedure():
    n_env, n_clips = 8, 20
    agent, task = _make_agent(True, n_env, n_clips)
    info, rec, failed = _spy_eval(agent, task)
    assert set(info) == KEYS8 and task._eval_mode is False
    term, _, pred_all, gt_all, batches = _reference_procedure(rec, n_env, n_clips)
    assert batches == 3                                        # 20 clips, 8 at a time: the last batch wraps around
    assert term.any() and (~term).any(), term                  # both failed and successful clips
    exp = EO.eval_info(pred_all, gt_all, term)
    # the success rate is the one the default path has always returned (a float32 mean of the termination flags)
    assert info["eval/success_rate"] == float(1.0 - torch.from_numpy(term).float().mean())
    assert abs(info["eval/success_rate"] - exp["eval/success_rate"]) < 1e-6
    for k in KEYS8 - {"eval/success_rate"}:
        assert np.isfinite(exp[k]), k
        assert abs(info[k] - exp[k]) <= 1e-3 + 1e-4 * abs(exp[k]), (k, info[k], exp[k])
    # frame weighting differs from the clip-weighted default
    per_clip = [np.linalg.norm(p - g, axis=-1).mean() * 1000 for p, g in zip(pred_all, gt_all) if len(p)]
    assert abs(info["eval/mpjpe_all"] - float(np.mean(per_clip))) > 1e-3
    # the failed keys update_training_data receives are those of the terminated clips
    keys = np.asarray(task._motion_data._motion_data_keys)
    assert failed == keys[term].tolist() and len(agent._metric_rows) == 3


def test_im_amp_default_eval_keeps_the_three_keys_and_two_sweeps_are_identical():
    n_env, n_clips = 8, 20
    agent, task = _make_agent(False, n_env, n_clips)
    info, rec, failed = _spy_eval(agent, task)
    assert set(info) == {"eval/success_rate", "eval/mpjpe_all", "eval/mpjpe_succ"}
    term, per_clip, _, _, _ = _reference_procedure(rec, n_env, n_clips)
    assert term.any() and (~term).any()
    assert failed == np.asarray(task._motion_data._motion_data_keys)[term].tolist()
    assert abs(info["eval/success_rate"] - float(1 - term.mean())) < 1e-6
    m_all, m_succ = float(per_clip.mean()) * 1000, float(per_clip[torch.from_numpy(~term)].mean()) * 1000
    assert abs(info["eval/mpjpe_all"] - m_all) < 1e-3 + 1e-4 * m_all
    assert abs(info["eval/mpjpe_succ"] - m_succ) < 1e-3 + 1e-4 * m_succ
    # the option on, the same seeded setup built twice: the same dict bit for bit.  (Two sweeps of ONE task differ in the last bits:
    # every sweep reloads its clips with new random headings, so the second sees the same errors between rotated positions.)
    a = _make_agent(True, n_env, n_clips)[0].eval()
    b = _make_agent(True, n_env, n_clips)[0].eval()
    assert set(a) == KEYS8 and a == b
    assert a["eval/success_rate"] == info["eval/success_rate"]
