"""GPU tests of the get-up schedule (HumanoidImGetup / HumanoidImMCPGetup): the recovery step launch (PHC_FLAG_RECOVERY) against the
plain launch plus the restated override (tests/getup_sched_oracle.py), the AMP vector of the current state (PHC_FLAG_AMP_CURRENT)
against the step's own row, the reset selection (phc_getup_reset) bit for bit against the oracle, and the task / agent on SyntheticSim."""
import pytest
import torch

from tests.getup_sched_oracle import recovery_step, reset_select
from phc_b200 import _lib, ops, synthetic as syn
from tests.helpers import close
from phc_b200.env.humanoid_im import RLGPUEnv
from phc_b200.env.humanoid_im_getup import HumanoidImGetup, HumanoidImMCPGetup
from phc_b200.learning.amp_agent import AMPAgent

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _setup(kind, n, seed):
    if kind == "j20":         # a spherical-joint humanoid of another body count: the generic (run-time J) instantiation
        m = syn.make_motions(max(1, n // 3), seed=seed, num_bodies=20, min_frames=20, max_frames=40)
        cfg = ops.EnvStepConfig(key_bodies=[19, 12], reset_bodies=None, dof_subset=None)
        st = syn.make_env_state(m, n, seed=seed, amp_dim=13 + 9 * 19 + 3 * 2, max_progress=40)
    elif kind == "smplx":
        m = syn.make_motions(max(1, n // 3), seed=seed, num_bodies=52, min_frames=20, max_frames=40)
        cfg = ops.EnvStepConfig(key_bodies=syn.SMPLX_KEY_BODIES, reset_bodies=None, dof_subset=None)
        st = syn.make_env_state(m, n, seed=seed, amp_dim=13 + 9 * 51 + 3 * len(syn.SMPLX_KEY_BODIES), max_progress=40)
    else:
        m = syn.make_motions(max(1, n // 3), seed=seed, min_frames=20, max_frames=40)
        kw = dict(obs_v=7) if kind == "kp" else {}
        if kind == "getup":
            kw = dict(zero_out_far=True)
        cfg = ops.EnvStepConfig(key_bodies=syn.SMPL_KEY_BODIES, reset_bodies=syn.SMPL_RESET_BODIES, dof_subset=syn.SMPL_DOF_SUBSET, **kw)
        st = syn.make_env_state(m, n, seed=seed, max_progress=40)
    d, s = m.to(DEV), st.to(DEV)
    mlib = ops.pack_motion_lib(d.gts, d.grs, d.gvs, d.gavs, d.lrs, d.dvs, d.lengths, d.num_frames, d.dts, d.length_starts)
    return mlib, cfg, s


def _plan(mlib, cfg, s, progress, cache, point_goal, **kw):
    return ops.EnvStepPlan(cfg, mlib, s.body_state, s.dof_state, s.dof_force, progress, s.motion_ids, s.start_times.clone(),
                           s.start_offsets.clone(), s.global_offset.clone(), amp_obs_buf=torch.zeros_like(s.amp_hist), amp_shift=False,
                           ref_cache=cache, reward_from_cache=cache is not None, point_goal=point_goal, **kw)


@pytest.mark.parametrize("kind", ["smpl", "getup", "kp", "j20", "smplx"])
@pytest.mark.parametrize("n", [3, 257, 4096, 16384])
def test_recovery_step_is_the_plain_step_with_the_override(kind, n):
    """A recovery launch = the plain launch at `progress` for reward / reset / AMP, the override of humanoid_im_getup.py:203-210, and for
    the still-recovering envs the observation and pose cache of the plain launch at `progress - 1` (the reference observes after the
    decrement).  Integers exact, floats bit for bit."""
    mlib, cfg, s = _setup(kind, n, seed=n % 97)
    g = torch.Generator(device=DEV).manual_seed(n)
    counter0 = torch.randint(0, 4, (n,), generator=g, device=DEV, dtype=torch.int32)
    counter0[: max(1, n // 4)] = 0
    p = s.progress.clone()
    bs = int(mlib.frames_body.shape[1])
    cache0 = torch.randn(n, bs, generator=g, device=DEV)
    pg0 = torch.rand(n, generator=g, device=DEV)
    # the two launches the recovery launch is made of: the same instantiation with idle counters at `progress` and at the decremented
    # progress (each reads the same cached pose), and the plain kernel, which has to agree with the idle recovery launch at the parity
    # tolerance (a separate template instantiation), integers exactly
    outs = []
    for prog in (p, torch.where(counter0 > 1, p - 1, p), p):
        cache = cache0.clone()
        plan = _plan(mlib, cfg, s, prog.clone(), cache, pg0.clone() if kind == "getup" else None)
        if len(outs) < 2:
            plan.set_recovery_counter(torch.zeros(n, dtype=torch.int32, device=DEV))
        plan.run()
        outs.append((plan, cache))
    (A, cache_a), (B, cache_b), (P, _) = outs
    for k in ("obs", "rew", "reward_raw", "amp_obs_buf"):
        close(getattr(A, k).cpu(), getattr(P, k).cpu(), what=f"idle recovery launch vs plain launch: {k}")
    assert torch.equal(A.reset, P.reset) and torch.equal(A.terminate, P.terminate)
    cache = cache0.clone()
    counter = counter0.clone()
    prog = p.clone()
    R = _plan(mlib, cfg, s, prog, cache, pg0.clone() if kind == "getup" else None)
    R.set_recovery_counter(counter)
    R.run()
    torch.cuda.synchronize()
    c_exp, p_exp, r_exp, t_exp, rec = recovery_step(counter0, p, A.reset, A.terminate)
    assert torch.equal(counter, c_exp) and torch.equal(prog, p_exp)
    assert torch.equal(R.reset, r_exp) and torch.equal(R.terminate, t_exp)
    assert torch.equal(R.rew, A.rew) and torch.equal(R.reward_raw, A.reward_raw)
    assert torch.equal(R.amp_obs_buf[:, 0], A.amp_obs_buf[:, 0])
    r2 = rec.unsqueeze(1)
    assert torch.equal(R.obs, torch.where(r2, B.obs, A.obs))
    assert torch.equal(cache, torch.where(r2, cache_b, cache_a))
    if n >= 257:
        assert rec.any() and (~rec).any()


@pytest.mark.parametrize("kind", ["smpl", "getup", "kp", "j20", "smplx"])
def test_amp_of_current_state_equals_the_step_row(kind):
    """PHC_FLAG_AMP_CURRENT on the observation-only launch writes, for the masked envs only, the AMP row the fused get-up step launch
    writes for the same simulator state (torch.equal), and the same observation row as the plain observation-only launch (parity
    tolerance: another instantiation)."""
    n = 1000
    mlib, cfg, s = _setup(kind, n, seed=4)
    step = _plan(mlib, cfg, s, s.progress.clone(), None, torch.zeros(n, device=DEV) if kind == "getup" else None)
    step.set_recovery_counter(torch.zeros(n, dtype=torch.int32, device=DEV))      # the get-up step launch
    step.run()
    mask = (torch.arange(n, device=DEV) % 3 == 1).long()
    amp = torch.full_like(s.amp_hist, -7.0)
    kw = dict(point_goal=torch.zeros(n, device=DEV)) if kind == "getup" else {}
    common = (cfg, mlib, s.body_state, s.dof_state, s.dof_force, s.progress, s.motion_ids, s.start_times, s.start_offsets, s.global_offset)
    cur = ops.EnvStepPlan(*common, only_where=mask, obs_only=True, amp_obs_buf=amp, amp_current=True, **kw)
    plain = ops.EnvStepPlan(*common, only_where=mask, obs_only=True, with_amp=False, **kw)
    cur.run()
    plain.run()
    torch.cuda.synchronize()
    m = mask.bool()
    assert torch.equal(amp[m, 0], step.amp_obs_buf[m, 0])
    assert (amp[~m] == -7.0).all() and (amp[m, 1:] == -7.0).all()
    close(cur.obs[m].cpu(), plain.obs[m].cpu(), what="observation of the AMP_CURRENT launch")


def _select_inputs(n, seed, D, bpe=24):
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = lambda *sh: torch.rand(*sh, generator=g, device=DEV)
    mask = (r(n) < 0.4).long()
    terminate = (r(n) < 0.5).long()
    perm = torch.argsort(r(n))
    available = (r(n) < 0.3).long()
    assignment = torch.randint(0, n, (n,), generator=g, device=DEV)     # stale / shared assignments included
    # no env holds more than one mark and marked states are held by non-resetting envs, as the schedule guarantees
    held = torch.zeros(n, dtype=torch.long, device=DEV)
    keep = (mask == 0) & (r(n) < 0.3)
    held[assignment[keep]] = 1
    available = held
    return dict(mask=mask, terminate=terminate, u_rec=r(n), u_fall=r(n), perm=perm, available=available, assignment=assignment,
                counter=torch.randint(0, 90, (n,), generator=g, device=DEV, dtype=torch.int32),
                body_state=torch.randn(n, bpe, 13, generator=g, device=DEV), dof_state=torch.randn(n, D, 2, generator=g, device=DEV),
                progress=torch.randint(0, 300, (n,), generator=g, device=DEV), reset=(r(n) < 0.5).long(), term=terminate.clone(),
                fall_root=torch.randn(n, 13, generator=g, device=DEV), fall_dof=torch.randn(n, D, generator=g, device=DEV))


@pytest.mark.parametrize("n", [3, 257, 4096, 16384])
@pytest.mark.parametrize("probs", [(0.0, 1.0), (0.5, 0.3), (1.0, 0.0)])
def test_reset_selection_matches_the_oracle_bit_for_bit(n, probs):
    """phc_getup_reset against the restated _reset_actors: both schedule phases (p_rec 0 / p_fall 1 before getup_udpate_epoch, the
    configured 0.5 / 0.3 after), mixed terminated envs, stale assignments; every output exact; distinct fall states within the reset."""
    D = 69
    x = _select_inputs(n, seed=n + int(probs[0] * 10), D=D)
    p_rec, p_fall = probs
    exp = reset_select(*(x[k].cpu() for k in ("mask", "terminate", "u_rec", "u_fall", "perm")), p_rec, p_fall, 90,
                       x["fall_root"].cpu(), x["fall_dof"].cpu(), *(x[k].cpu() for k in ("available", "assignment", "counter", "body_state",
                                                                                          "dof_state", "progress", "reset", "term")))
    ref_init, fall = torch.zeros(n, dtype=torch.long, device=DEV), torch.zeros(n, dtype=torch.long, device=DEV)
    pd = torch.tensor([p_rec, p_fall], device=DEV)
    ops.getup_reset(x["mask"], x["term"], x["u_rec"], x["u_fall"], x["perm"], pd[0:1], pd[1:2], 90, x["fall_root"], x["fall_dof"],
                    x["available"], x["assignment"], x["counter"], x["body_state"], x["dof_state"], x["progress"], x["reset"], x["term"],
                    ref_init, fall)
    torch.cuda.synchronize()
    got = dict(available=x["available"], assignment=x["assignment"], counter=x["counter"], body_state=x["body_state"],
               dof_state=x["dof_state"], progress=x["progress"], reset=x["reset"], terminate=x["term"], ref_init=ref_init, fall=fall)
    for k, v in exp.items():
        assert torch.equal(got[k].cpu(), v), f"{k} differs (n={n}, probs={probs})"
    fs = got["assignment"][fall.bool()]
    assert fs.unique().numel() == fs.numel()
    if n >= 257 and p_fall > 0:
        assert fall.sum() > 0


def test_reset_selection_refuses_a_bank_of_the_wrong_size():
    n = 8
    x = _select_inputs(n, 0, D=69)
    pd = torch.tensor([0.5, 0.5], device=DEV)
    with pytest.raises(_lib.PhcError, match="num_states"):
        ops.getup_reset(x["mask"], x["term"], x["u_rec"], x["u_fall"], x["perm"][:4], pd[0:1], pd[1:2], 90, x["fall_root"][:4],
                        x["fall_dof"][:4], x["available"][:4], x["assignment"], x["counter"], x["body_state"], x["dof_state"], x["progress"],
                        x["reset"], x["term"], torch.zeros_like(x["mask"]), torch.zeros_like(x["mask"]))


GETUP_ENV = {"recoveryEpisodeProb": 0.5, "recoverySteps": 90, "fallInitProb": 0.3, "getup_schedule": True, "getup_udpate_epoch": 2}


def _getup_task(n, seed=0, cls=HumanoidImGetup, **kw):
    m = syn.make_motions(max(1, n // 4), seed=seed, min_frames=20, max_frames=40)
    env = dict(GETUP_ENV, num_envs=n, episode_length=60)
    env.update(kw.pop("env", {}))
    return cls({"env": env, "motion_data": m, "seed": seed, **kw})


def _run_task(task, steps, seed):
    torch.manual_seed(seed)
    task.update_getup_schedule(5, getup_udpate_epoch=2)          # the configured probabilities
    task.reset()
    N = task.num_envs
    hist = []
    for t in range(steps):
        task.reset(task.reset_buf.clone())
        c0, p0 = task._recovery_counter.clone(), task.progress_buf.clone()
        task.step(torch.zeros(N, task.num_dof, device=task.device))
        c1 = task._recovery_counter
        rec = c1 > 0
        assert torch.equal(c1, torch.clamp_min(c0 - 1, 0))
        assert (task.reset_buf[rec] == 0).all() and (task._terminate_buf[rec] == 0).all(), "a recovering env reset"
        assert torch.equal(task.progress_buf[rec], p0[rec]), "progress advanced while the counter ran"
        hist.append((task.obs_buf.clone(), task.rew_buf.clone(), task.reset_buf.clone(), c1.clone(), task.progress_buf.clone(),
                     task._amp_obs_buf.clone()))
    return hist


def test_getup_task_on_synthetic_sim_for_200_steps_and_cache_bit_identity():
    """HumanoidImGetup on SyntheticSim: recovering envs never reset, their progress stays frozen while the counter runs; fall starts
    and recoveries both happen; the run is bit-identical with the pose cache on and off."""
    runs = []
    for cache in (True, False):
        task = _getup_task(512, seed=3, ref_pose_cache=cache, specialised_step=False)
        runs.append(_run_task(task, 200, seed=11))
        assert int(task.availalbe_fall_states.sum()) > 0
    seen_rec = any(bool((h[3] > 0).any()) for h in runs[0])
    assert seen_rec
    for t, (a, b) in enumerate(zip(*runs)):
        for i, (x, y) in enumerate(zip(a, b)):
            assert torch.equal(x, y), f"step {t}: output {i} differs between pose cache on and off"


def test_fall_start_amp_history_is_the_current_state_in_every_slot():
    task = _getup_task(256, seed=1)
    task.update_getup_schedule(0, getup_udpate_epoch=2)          # before the switch: every reset is a fall start
    torch.manual_seed(0)
    task.reset()
    torch.cuda.synchronize()
    assert task._fall_mask.all() and not task._ref_init_mask.any()
    w = task._amp_obs_buf
    assert torch.equal(w, w[:, :1].expand_as(w))
    assert torch.equal(task._rigid_body_state_reshaped[:, 0], task._fall_root_states[task.fall_id_assignments])
    assert (task._recovery_counter == 90).all() and (task.progress_buf == 0).all()


def test_missing_backend_hook_is_refused():
    from phc_b200.env.humanoid_im import SyntheticSim
    m = syn.make_motions(4, seed=0, min_frames=20, max_frames=40)
    sim = SyntheticSim(m, 8, DEV)

    class Plain:                      # a complete backend except for generate_fall_states
        graph_safe = True

        def __init__(self, s):
            self.rigid_body_state, self.dof_state, self.dof_force, self.bodies_per_env = s.rigid_body_state, s.dof_state, s.dof_force, s.bodies_per_env

        def set_env_state(self, *a):
            pass

        def simulate(self, a):
            pass
    with pytest.raises(TypeError, match="generate_fall_states"):
        HumanoidImGetup({"env": dict(GETUP_ENV, num_envs=8), "motion_data": m, "sim_backend": Plain(sim)})


def test_agent_across_the_switch_epoch_graph_equals_eager():
    """AMPAgent with the get-up schedule (getup_udpate_epoch 2): the reward weights switch from (0, 1) to (0.5, 0.5) after epoch 2, the
    task's probabilities follow, and the graph-replayed rollout equals the eager one bit for bit across the switch."""
    n = 96
    cfgs = {"horizon_length": 8, "minibatch_size": 256, "amp_minibatch_size": 64, "mini_epochs": 1, "amp_obs_demo_buffer_size": 1024,
            "amp_replay_buffer_size": 1024, "amp_batch_size": 128,
            "network": {"mlp": {"units": [64, 32], "activation": "relu"}, "disc": {"units": [64, 32], "activation": "relu"}}}
    agents = []
    for graphed in (False, True):
        task = _getup_task(n, seed=5)
        torch.manual_seed(1234)
        ag = AMPAgent("t", dict(cfgs, vec_env=RLGPUEnv(task), graph_rollout=graphed))
        ag.obs = ag.env_reset()
        ag._init_amp_demo_buf()
        agents.append(ag)
    for epoch in range(5):
        outs = []
        for ag in agents:
            ag.pre_epoch(epoch)
            task = ag.vec_env.env.task
            if epoch > 2:
                assert (ag._task_reward_w, ag._disc_reward_w) == (0.5, 0.5) and (task._recovery_episode_prob, task._fall_init_prob) == (0.5, 0.3)
            else:
                assert (ag._task_reward_w, ag._disc_reward_w) == (0, 1) and (task._recovery_episode_prob, task._fall_init_prob) == (0, 1)
            torch.manual_seed(77 + epoch)
            ag.set_eval()
            bd = ag.play_steps()
            torch.cuda.synchronize()
            outs.append({k: v.clone() for k, v in ag.experience_buffer.items()} | {"mb_rewards": bd["mb_rewards"].clone(),
                                                                                    "counter": task._recovery_counter.clone()})
        for k in outs[0]:
            assert torch.equal(outs[0][k], outs[1][k]), f"epoch {epoch}: {k} differs between the eager and the graph-replayed rollout"
    assert agents[1]._rollout_graph is not None


def _pnn_checkpoint(obs_dim, act_dim, K, units=(64, 32), seed=0):
    """A frozen-primitive checkpoint in the layout HumanoidImMCP loads (as test_gpu_mcp.py builds one)."""
    gen = torch.Generator().manual_seed(seed)
    sd = {}
    for k in range(K):
        d = obs_dim
        for i, u in enumerate(list(units) + [act_dim]):
            sd[f"a2c_network.pnn.actors.{k}.{2 * i}.weight"] = torch.randn(u, d, generator=gen) / d ** 0.5
            sd[f"a2c_network.pnn.actors.{k}.{2 * i}.bias"] = torch.randn(u, generator=gen) * 0.1
            d = u
    sd["a2c_network.mu.bias"] = torch.zeros(act_dim)
    rms = {"running_mean": torch.randn(obs_dim, generator=gen, dtype=torch.float64) * 0.1,
           "running_var": torch.rand(obs_dim, generator=gen, dtype=torch.float64) + 0.5}
    return {"model": sd, "running_mean_std": rms}


def test_mcp_getup_with_a_pnn_checkpoint():
    """HumanoidImMCPGetup: the composer task (frozen PNN primitives) with the get-up schedule; steps with mixed weights keep the
    recovery invariants."""
    n, K = 64, 3
    m = syn.make_motions(16, seed=2, min_frames=20, max_frames=40)
    probe = HumanoidImGetup({"env": dict(GETUP_ENV, num_envs=n), "motion_data": m, "seed": 2})
    ck = _pnn_checkpoint(probe.get_obs_size(), probe.num_dof, K)
    del probe
    task = HumanoidImMCPGetup({"env": dict(GETUP_ENV, num_envs=n, num_prim=K, has_pnn=True, has_lateral=False), "motion_data": m, "seed": 2},
                              pnn_checkpoint=ck)
    assert task.get_action_size() == K and task.getup_schedule
    task.update_getup_schedule(5, getup_udpate_epoch=2)
    torch.manual_seed(0)
    task.reset()
    for _ in range(20):
        task.reset(task.reset_buf.clone())
        p0 = task.progress_buf.clone()
        task.step(torch.rand(n, K, device=DEV))
        rec = task._recovery_counter > 0
        assert (task.reset_buf[rec] == 0).all() and torch.equal(task.progress_buf[rec], p0[rec])
    assert torch.isfinite(task.obs_buf).all()


def test_eval_zeroes_and_restores_the_probabilities():
    from phc_b200.learning.im_amp import IMAmpAgent
    task = _getup_task(32, seed=0)
    task.update_getup_schedule(5, getup_udpate_epoch=2)
    seen = {}

    class Stop(Exception):
        pass

    def spy_mode(on):
        pass

    def spy_begin():                   # the sweep's first reset: record what the task sees
        seen["probs"] = (task._recovery_episode_prob, task._fall_init_prob, float(task._p_dev[0]), float(task._p_dev[1]))

    def stop(*a):                      # ... and stop at the first step of the sweep
        raise Stop()
    task.set_eval_mode = spy_mode
    task.begin_seq_motion_samples = spy_begin
    task._motion_data.load_motions = lambda **kw: None        # eval walks a loadable library; the spy stops it before any load
    task.resample_motions = lambda: None
    ag = IMAmpAgent.__new__(IMAmpAgent)
    ag.vec_env = RLGPUEnv(task)
    ag.device = task.device
    ag.set_eval = lambda: None
    ag.env_reset = stop
    with pytest.raises(Stop):
        ag.eval()
    assert seen["probs"] == (0.0, 0.0, 0.0, 0.0)
    assert (task._recovery_episode_prob, task._fall_init_prob) == (0.5, 0.3)
    assert torch.equal(task._p_dev.cpu(), torch.tensor([0.5, 0.3]))


def test_probabilities_reach_the_device():
    """set_getup_probs writes the device copy the selection reads; a plain assignment to the attributes (the reference's own eval does
    that) reaches it at the next reset."""
    task = _getup_task(64, seed=0)
    task.set_getup_probs(0.25, 0.75)
    assert torch.equal(task._p_dev.cpu(), torch.tensor([0.25, 0.75]))
    task._recovery_episode_prob, task._fall_init_prob = 0, 0
    torch.manual_seed(0)
    task.reset()
    torch.cuda.synchronize()
    assert torch.equal(task._p_dev.cpu(), torch.zeros(2)) and not task._fall_mask.any()


def test_env_step_refusals_of_the_getup_flags():
    """PHC_ERR_INVALID_ARG for the flag on the observation-only launch, a NULL counter or PHC_FLAG_AMP_CURRENT on a step launch;
    PHC_ERR_UNSUPPORTED for time_steps > 1 and for the keypoint observation on a body count other than 24.  Refused before any launch."""
    lib = _lib.load()
    mlib, cfg, s = _setup("smpl", 16, seed=0)
    plan = _plan(mlib, cfg, s, s.progress.clone(), None, None)
    counter = torch.zeros(16, dtype=torch.int32, device=DEV)
    a = plan.args
    base = a.flags

    def rc(flags, **fields):
        saved = {k: getattr(a, k) for k in fields}
        a.flags = flags
        for k, v in fields.items():
            setattr(a, k, v)
        try:
            return lib.phc_env_step(plan._args_ref, ops._stream())
        finally:
            a.flags = base
            for k, v in saved.items():
                setattr(a, k, v)
    R, AC, OO = _lib.PHC_FLAG_RECOVERY, _lib.PHC_FLAG_AMP_CURRENT, _lib.PHC_FLAG_OBS_ONLY
    assert rc(base | R | OO, recovery_counter=counter.data_ptr()) == -1
    assert "observation-only" in lib.phc_last_error().decode()
    assert rc(base | R, recovery_counter=None) == -1
    assert rc(base | AC) == -1
    assert rc(base | R, recovery_counter=counter.data_ptr(), time_steps=2, traj_dt=1.0 / 30) == -2
    assert "time_steps 1" in lib.phc_last_error().decode()
    # a hinge-joint robot (num_dofs > 0) and extend bodies are refused the same way, before any launch
    lc = a.lib
    saved = (lc.num_dofs, lc.num_ext_bodies, lc.body_stride)
    try:
        lc.num_dofs = 23
        a.lib = lc
        assert rc(base | R, recovery_counter=counter.data_ptr()) == -2 and "spherical-joint" in lib.phc_last_error().decode()
        assert rc(base | OO | AC) == -2
        lc.num_dofs, lc.num_ext_bodies, lc.body_stride = 0, 1, lib.phc_motion_body_stride(25)
        a.lib = lc
        assert rc(base | R, recovery_counter=counter.data_ptr()) == -2 and "extend bodies" in lib.phc_last_error().decode()
    finally:
        lc.num_dofs, lc.num_ext_bodies, lc.body_stride = saved
        a.lib = lc
    torch.cuda.synchronize()
    assert torch.equal(counter, torch.zeros_like(counter))            # nothing ran


# ---- the C ABI against tests/golden/getup_sched.npz (the unmodified reference, make_golden_getup_sched.py) ---------------------------
from tests.getup_sched_cases import RESETS, STEPS, load as load_golden, prefixed, source  # noqa: E402

GS = load_golden("getup_sched.npz")


def _golden_cfg(J):
    if J == "24":
        return ops.EnvStepConfig(key_bodies=syn.SMPL_KEY_BODIES, reset_bodies=syn.SMPL_RESET_BODIES, dof_subset=syn.SMPL_DOF_SUBSET,
                                 zero_out_far=True, cycle_motion=True, max_episode_length=15)
    return ops.EnvStepConfig(key_bodies=syn.SMPLX_KEY_BODIES, reset_bodies=None, dof_subset=None, zero_out_far=True, cycle_motion=True,
                             max_episode_length=15)


def _golden_env(J):
    g, m, st = source(J)
    d, s = m.to(DEV), st.to(DEV)
    mlib = ops.pack_motion_lib(d.gts, d.grs, d.gvs, d.gavs, d.lrs, d.dvs, d.lengths, d.num_frames, d.dts, d.length_starts)
    extra = dict(point_goal=g["in_point_goal"].to(DEV).clone(), cycle_counter=g["in_cycle_counter"].to(DEV, torch.int32).clone(),
                 cycle_phase=torch.zeros(s.progress.shape[0], device=DEV))
    return mlib, s, extra


@pytest.mark.parametrize("J", ["24", "52"])
def test_recovery_steps_c_abi_vs_reference_golden(J):
    """Three recovery step launches (SMPL: the GETUP recovery instantiation; SMPL-X: the strided kernel) against the reference's
    HumanoidImGetup steps: counters, progress decrement, the override under cycle_motion / pass_time, integers exact."""
    mlib, s, extra = _golden_env(J)
    plan = ops.EnvStepPlan(_golden_cfg(J), mlib, s.body_state, s.dof_state, s.dof_force, s.progress, s.motion_ids, s.start_times,
                           s.start_offsets, s.global_offset, amp_obs_buf=s.amp_hist.clone(), **extra)
    rc = GS[f"step{J}_in_recovery_counter"].to(DEV, torch.int32).clone()
    plan.set_recovery_counter(rc)
    for k in range(STEPS):
        e = prefixed(GS, f"step{J}_{k}_")
        if k > 0:
            s.progress += 1
        extra["cycle_phase"].copy_(e["in_cycle_phase"])
        plan.run()
        torch.cuda.synchronize()
        got = dict(reset=plan.reset, terminate=plan.terminate, progress=s.progress, recovery_counter=rc, cycle_counter=extra["cycle_counter"],
                   rew=plan.rew, reward_raw=plan.reward_raw, start_times=s.start_times, start_offsets=s.start_offsets,
                   global_offset=s.global_offset, point_goal=extra["point_goal"])
        for name in ("reset", "terminate", "progress", "recovery_counter", "cycle_counter"):
            assert torch.equal(got[name].cpu().to(e["out_" + name].dtype), e["out_" + name]), f"step {k}: {name}"
        for name in ("rew", "reward_raw", "start_times", "start_offsets", "global_offset", "point_goal"):
            close(got[name].cpu(), e["out_" + name], what=f"step {k}: {name}")
        close(plan.obs.cpu()[e["out_obs_rows"]], e["out_obs"], rtol=1e-5, atol=2e-6, what=f"step {k}: obs of the recovering envs")


@pytest.mark.parametrize("J", ["24", "52"])
def test_reset_selection_c_abi_vs_reference_golden(J):
    """Four resets through phc_getup_reset + the observation-only launch with PHC_FLAG_AMP_CURRENT + phc_amp_ring_fill against the
    reference's _reset_actors / _compute_observations(env_ids) / _init_amp_obs: selection, bank, counters and fall states exact;
    observation rows and AMP history of the fall and recovery envs at the parity tolerance."""
    mlib, s, extra = _golden_env(J)
    N, D = s.body_state.shape[0], s.dof_state.shape[1]
    amp = s.amp_hist.clone()
    mask = torch.zeros(N, dtype=torch.long, device=DEV)
    plan = ops.EnvStepPlan(_golden_cfg(J), mlib, s.body_state, s.dof_state, s.dof_force, s.progress, s.motion_ids, s.start_times,
                           s.start_offsets, s.global_offset, only_where=mask, obs_only=True, amp_obs_buf=amp, amp_current=True, **extra)
    fall_root, fall_dof = GS[f"sel{J}_fall_root"].to(DEV), GS[f"sel{J}_fall_dof_pos"].to(DEV)
    available, assignment = torch.zeros(N, dtype=torch.long, device=DEV), torch.zeros(N, dtype=torch.long, device=DEV)
    counter = torch.zeros(N, dtype=torch.int32, device=DEV)
    reset, term = torch.zeros(N, dtype=torch.long, device=DEV), torch.zeros(N, dtype=torch.long, device=DEV)
    ref_init, fall = torch.zeros_like(reset), torch.zeros_like(reset)
    for r in range(RESETS):
        e = {k: v.to(DEV) for k, v in prefixed(GS, f"sel{J}_{r}_").items()}
        mask.copy_(e["in_mask"]); s.progress.copy_(e["in_progress"]); reset.copy_(e["in_reset"]); term.copy_(e["in_terminate"])
        ops.getup_reset(mask, term, e["in_u_rec"], e["in_u_fall"], e["in_perm"], e["in_probs"][0:1], e["in_probs"][1:2], 90, fall_root,
                        fall_dof, available, assignment, counter, s.body_state, s.dof_state, s.progress, reset, term, ref_init, fall)
        plan.run()
        ops.amp_ring_fill(amp, None, fall)
        torch.cuda.synchronize()
        for name, v in (("available", available), ("assignment", assignment), ("ref_init", ref_init), ("fall", fall)):
            assert torch.equal(v, e["out_" + name]), f"reset {r}: {name}"
        assert torch.equal(counter, e["out_recovery_counter"].to(torch.int32)), f"reset {r}: counter"
        rows = e["out_rows"]
        for name, v in (("progress", s.progress), ("reset", reset), ("terminate", term)):
            assert torch.equal(v[rows], e["out_" + name][rows]), f"reset {r}: {name}"
        assert torch.equal(s.body_state[:, 0], e["out_root_state"]) and torch.equal(s.dof_state[..., 0], e["out_dof_pos"])
        assert (s.dof_state[fall.bool(), :, 1] == 0).all()
        if "out_obs" in e:
            close(plan.obs[rows].cpu(), e["out_obs"].cpu(), rtol=1e-5, atol=2e-6, what=f"reset {r}: obs")
        close(amp[rows, 0].cpu(), e["out_amp_newest"].cpu(), rtol=1e-5, atol=2e-6, what=f"reset {r}: newest AMP slot")
        f = fall.bool()
        assert torch.equal(amp[f], amp[f, :1].expand_as(amp[f]))
