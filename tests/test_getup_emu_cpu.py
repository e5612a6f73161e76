"""The get-up schedule's kernel code on the CPU: the recovery instantiations of env_step_kernel (SMPL, generic run-time J, keypoint)
and of the strided kernel, phc_getup_reset's selection and copy kernels and phc_amp_ring_fill, through the emulation of tests/emu
(verbatim product source; the selection runs as one block of 1024 concurrent threads), with arguments assembled by ops.EnvStepPlan on
host tensors.  Against tests/golden/getup_sched.npz from the unmodified reference and against tests/getup_sched_oracle.py; one subset
again with every lane dawdling after each collective (PHC_EMU_CHAOS=1)."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

from phc_b200 import ops, synthetic as syn                                   # noqa: E402
from tests.getup_sched_cases import RESETS, STEPS, load, prefixed, source    # noqa: E402
from tests.getup_sched_oracle import reset_select                           # noqa: E402
from tests.helpers import close                                              # noqa: E402

G = load("getup_sched.npz")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    import shutil
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    import getup_emu
    import host_plan
    return getup_emu.EmuGetup(getup_emu.build(str(tmp_path_factory.mktemp("emu_getup")))), host_plan


def cfg_for(J, **kw):
    if J == "24":
        return ops.EnvStepConfig(key_bodies=syn.SMPL_KEY_BODIES, reset_bodies=syn.SMPL_RESET_BODIES, dof_subset=syn.SMPL_DOF_SUBSET,
                                 zero_out_far=True, cycle_motion=True, max_episode_length=15, **kw)
    return ops.EnvStepConfig(key_bodies=syn.SMPLX_KEY_BODIES, reset_bodies=None, dof_subset=None, zero_out_far=True, cycle_motion=True,
                             max_episode_length=15, **kw)


def host_plan_for(hp, J, m, st, g, cfg, **kw):
    mlib = hp.host_pack(m.gts, m.grs, m.gvs, m.gavs, m.lengths, m.num_frames, m.dts, m.length_starts)
    extra = dict(point_goal=g["in_point_goal"].clone(), cycle_counter=g["in_cycle_counter"].to(torch.int32).clone(),
                 cycle_phase=torch.zeros(st.progress.shape[0]))
    with hp.host_mode():
        plan = ops.EnvStepPlan(cfg, mlib, st.body_state, st.dof_state, st.dof_force, st.progress, st.motion_ids, st.start_times,
                               st.start_offsets, st.global_offset, **extra, **kw)
    return plan, extra


@pytest.mark.parametrize("J,variant", [("24", "smpl"), ("24", "generic"), ("24", "kp"), ("52", "wide")])
def test_recovery_steps_vs_reference_golden(emu, J, variant):
    """Three recovery steps of every recovery instantiation against the reference's HumanoidImGetup steps (counters, progress decrement,
    the override under cycle_motion / pass_time exact; rewards and bookkeeping at the parity tolerance; the v6 observation rows of the
    recovering envs -- the keypoint instantiation writes v7 rows, whose arithmetic kp.npz pins)."""
    e_, hp = emu
    g, m, st = source(J)
    plan, extra = host_plan_for(hp, J, m, st, g, cfg_for(J, obs_v=7 if variant == "kp" else 6), amp_obs_buf=st.amp_hist.clone())
    rc = G[f"step{J}_in_recovery_counter"].to(torch.int32).clone()
    with hp.host_mode():
        plan.set_recovery_counter(rc)
    for k in range(STEPS):
        e = prefixed(G, f"step{J}_{k}_")
        if k > 0:
            st.progress += 1
        extra["cycle_phase"].copy_(e["in_cycle_phase"])
        e_.run(plan, variant)
        got = dict(reset=plan.reset, terminate=plan.terminate, progress=st.progress, recovery_counter=rc, cycle_counter=extra["cycle_counter"],
                   rew=plan.rew, reward_raw=plan.reward_raw, start_times=st.start_times, start_offsets=st.start_offsets,
                   global_offset=st.global_offset, point_goal=extra["point_goal"])
        for name in ("reset", "terminate", "progress", "recovery_counter", "cycle_counter"):
            assert torch.equal(got[name].to(e["out_" + name].dtype), e["out_" + name]), f"{variant} step {k}: {name}"
        for name in ("rew", "reward_raw", "start_times", "start_offsets", "global_offset", "point_goal"):
            close(got[name], e["out_" + name], what=f"{variant} step {k}: {name}")
        if variant != "kp":
            close(plan.obs[e["out_obs_rows"]], e["out_obs"], rtol=1e-5, atol=2e-6, what=f"{variant} step {k}: obs of the recovering envs")


@pytest.mark.parametrize("J,variant", [("24", "smpl"), ("52", "wide")])
def test_reset_path_vs_reference_golden(emu, J, variant):
    """Four resets: the emulated selection + copy kernels, the observation-only launch with PHC_FLAG_AMP_CURRENT and the ring fill
    against the reference's _reset_actors / _compute_observations(env_ids) / _init_amp_obs (bank, selection, counters, fall states
    exact; observation rows and AMP history of the fall and recovery envs at the parity tolerance)."""
    e_, hp = emu
    g, m, st = source(J)
    N = st.body_state.shape[0]
    amp = st.amp_hist.clone()
    mask = torch.zeros(N, dtype=torch.long)
    plan, _ = host_plan_for(hp, J, m, st, g, cfg_for(J), only_where=mask, obs_only=True, amp_obs_buf=amp, amp_current=True)
    fall_root, fall_dof = G[f"sel{J}_fall_root"].contiguous(), G[f"sel{J}_fall_dof_pos"].contiguous()
    available, assignment = torch.zeros(N, dtype=torch.long), torch.zeros(N, dtype=torch.long)
    counter = torch.zeros(N, dtype=torch.int32)
    reset, term, ref_init, fall = (torch.zeros(N, dtype=torch.long) for _ in range(4))
    for r in range(RESETS):
        e = prefixed(G, f"sel{J}_{r}_")
        mask.copy_(e["in_mask"]); st.progress.copy_(e["in_progress"]); reset.copy_(e["in_reset"]); term.copy_(e["in_terminate"])
        e_.getup_reset(mask, term, e["in_u_rec"].contiguous(), e["in_u_fall"].contiguous(), e["in_perm"].contiguous(), e["in_probs"].contiguous(),
                       90, fall_root, fall_dof, available, assignment, counter, st.body_state, st.dof_state, st.progress, reset, term, ref_init, fall)
        e_.run(plan, variant)
        e_.amp_ring_fill(amp, fall)
        for name, v in (("available", available), ("assignment", assignment), ("ref_init", ref_init), ("fall", fall)):
            assert torch.equal(v, e["out_" + name]), f"reset {r}: {name}"
        assert torch.equal(counter, e["out_recovery_counter"].to(torch.int32))
        rows = e["out_rows"]
        for name, v in (("progress", st.progress), ("reset", reset), ("terminate", term)):
            assert torch.equal(v[rows], e["out_" + name][rows]), f"reset {r}: {name}"
        assert torch.equal(st.body_state[:, 0], e["out_root_state"]) and torch.equal(st.dof_state[..., 0], e["out_dof_pos"])
        if "out_obs" in e:
            close(plan.obs[rows], e["out_obs"], rtol=1e-5, atol=2e-6, what=f"reset {r}: obs")
        close(amp[rows, 0], e["out_amp_newest"], rtol=1e-5, atol=2e-6, what=f"reset {r}: newest AMP slot")
        f = fall.bool()
        assert torch.equal(amp[f], amp[f, :1].expand_as(amp[f]))


@pytest.mark.parametrize("n,probs", [(2500, (0.5, 0.3)), (2500, (0.0, 1.0)), (1031, (1.0, 0.5))])
def test_selection_vs_oracle_across_chunks(emu, n, probs):
    """More envs than the selection CTA has threads (several scan chunks), stale and shared assignments: bit for bit against the oracle."""
    e_, _ = emu
    g = torch.Generator().manual_seed(n)
    r = lambda *sh: torch.rand(*sh, generator=g)
    D = 9
    mask, term = (r(n) < 0.4).long(), (r(n) < 0.5).long()
    assignment = torch.randint(0, n, (n,), generator=g)
    available = torch.zeros(n, dtype=torch.long)
    available[assignment[(mask == 0) & (r(n) < 0.3)]] = 1
    x = dict(u_rec=r(n), u_fall=r(n), perm=torch.argsort(r(n)), counter=torch.randint(0, 90, (n,), generator=g, dtype=torch.int32),
             body=torch.randn(n, 2, 13, generator=g), dof=torch.randn(n, D, 2, generator=g), progress=torch.randint(0, 300, (n,), generator=g),
             reset=(r(n) < 0.5).long(), fall_root=torch.randn(n, 13, generator=g), fall_dof=torch.randn(n, D, generator=g))
    exp = reset_select(mask, term, x["u_rec"], x["u_fall"], x["perm"], probs[0], probs[1], 90, x["fall_root"], x["fall_dof"], available,
                       assignment, x["counter"], x["body"], x["dof"], x["progress"], x["reset"], term)
    got = dict(available=available.clone(), assignment=assignment.clone(), counter=x["counter"].clone(), body_state=x["body"].clone(),
               dof_state=x["dof"].clone(), progress=x["progress"].clone(), reset=x["reset"].clone(), terminate=term.clone(),
               ref_init=torch.zeros(n, dtype=torch.long), fall=torch.zeros(n, dtype=torch.long))
    e_.getup_reset(mask, term.clone(), x["u_rec"], x["u_fall"], x["perm"], torch.tensor(probs, dtype=torch.float32), 90, x["fall_root"],
                   x["fall_dof"], got["available"], got["assignment"], got["counter"], got["body_state"], got["dof_state"], got["progress"],
                   got["reset"], got["terminate"], got["ref_init"], got["fall"])
    for k, v in exp.items():
        assert torch.equal(got[k], v), k
    assert int(got["fall"].sum()) > 0 or probs[1] == 0


def test_getup_chaos_mode_subset():
    """The same emulation with every lane dawdling randomly after each collective (PHC_EMU_CHAOS=1, read when the emulation library
    loads, hence a fresh process): the selection CTA's scans and phase barriers, and a recovery instantiation."""
    import subprocess
    if os.environ.get("PHC_EMU_CHAOS") == "1":
        pytest.skip("already inside the chaos run")
    env = dict(os.environ, PHC_EMU_CHAOS="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-p", "no:cacheprovider", "-k",
                        "reset_path and 24 or chunks and 1031 or golden and smpl"], capture_output=True, text=True, env=env,
                       cwd=os.path.dirname(HERE), timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
