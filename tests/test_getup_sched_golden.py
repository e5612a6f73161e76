"""The get-up schedule oracle (tests/getup_sched_oracle.py) against tests/golden/getup_sched.npz, produced by the unmodified reference
(tests/golden/make_golden_getup_sched.py): three env steps with recovery counters running down (cycle_motion wrap-around, pass_time,
early termination, the progress decrement) and four resets of a persistent fall-state bank in both schedule phases (stale
assignments included), at 24 (SMPL) and 52 (SMPL-X) bodies.  CPU only."""
import pytest
import torch

from tests.getup_sched_cases import RESETS, STEPS, load, prefixed, source
from tests.getup_sched_oracle import env_step_recovery, reset_select
from tests.helpers import close, oracle_tables, smpl_step_config
from oracle import phc_oracle as O
from phc_b200 import synthetic as syn

G = load("getup_sched.npz")


def step_config(J):
    if J == "24":
        return smpl_step_config()
    return O.StepConfig(key_bodies=syn.SMPLX_KEY_BODIES, reset_bodies=None, dof_subset=None)


@pytest.mark.parametrize("J", ["24", "52"])
def test_recovery_steps_oracle_vs_reference_golden(J):
    g, m, st = source(J)
    tab, cfg = oracle_tables(m), step_config(J)
    cc, pg, rc = g["in_cycle_counter"].clone(), g["in_point_goal"].clone(), G[f"step{J}_in_recovery_counter"].clone()
    prog, t0, t1, go, amp = st.progress.clone(), st.start_times.clone(), st.start_offsets.clone(), st.global_offset.clone(), st.amp_hist.clone()
    for k in range(STEPS):
        e = prefixed(G, f"step{J}_{k}_")
        if k > 0:
            prog = prog + 1
        out = env_step_recovery(tab, cfg, st.body_state, st.dof_state, st.dof_force, prog, st.motion_ids, t0, t1, go, amp, pg, cc,
                                e["in_cycle_phase"], rc, 15)
        for name in ("reset", "terminate", "progress", "recovery_counter", "cycle_counter"):
            assert torch.equal(out[name].to(e["out_" + name].dtype), e["out_" + name]), f"step {k}: {name}"
        for name in ("rew", "reward_raw", "start_times", "start_offsets", "global_offset", "point_goal"):
            close(out[name], e["out_" + name], what=f"step {k}: {name}")
        close(out["obs"][e["out_obs_rows"]], e["out_obs"], rtol=1e-5, atol=2e-6, what=f"step {k}: obs of the recovering envs")
        prog, rc, cc, pg = out["progress"], out["recovery_counter"], out["cycle_counter"], out["point_goal"]
        t0, t1, go, amp = out["start_times"], out["start_offsets"], out["global_offset"], out["amp_obs_buf"]
    assert int((rc == 0).sum()) > int((G[f"step{J}_in_recovery_counter"] == 0).sum())      # counters ran down


@pytest.mark.parametrize("J", ["24", "52"])
def test_reset_selection_oracle_vs_reference_golden(J):
    g, m, st = source(J)
    N, D = st.body_state.shape[0], st.dof_state.shape[1]
    fall_root, fall_dof = G[f"sel{J}_fall_root"], G[f"sel{J}_fall_dof_pos"]
    available, assignment = torch.zeros(N, dtype=torch.long), torch.zeros(N, dtype=torch.long)
    counter = torch.zeros(N, dtype=torch.int32)
    body, dof = st.body_state.clone(), st.dof_state.clone()
    for r in range(RESETS):
        e = prefixed(G, f"sel{J}_{r}_")
        p_rec, p_fall = e["in_probs"].tolist()
        out = reset_select(e["in_mask"], e["in_terminate"], e["in_u_rec"], e["in_u_fall"], e["in_perm"], torch.tensor(p_rec),
                           torch.tensor(p_fall), 90, fall_root, fall_dof, available, assignment, counter, body, dof, e["in_progress"],
                           e["in_reset"], e["in_terminate"])
        for name in ("available", "assignment", "ref_init", "fall"):
            assert torch.equal(out[name], e["out_" + name]), f"reset {r}: {name}"
        assert torch.equal(out["counter"], e["out_recovery_counter"].to(torch.int32)), f"reset {r}: counter"
        fr = (out["fall"] == 1) | ((e["in_mask"] == 1) & (out["ref_init"] == 0))        # fall + recovery envs (the reference zeroes
        for name in ("progress", "reset", "terminate"):                                    # ref-init envs in the same statement)
            assert torch.equal(out[name][fr], e["out_" + name][fr]), f"reset {r}: {name}"
        assert torch.equal(out["body_state"][:, 0], e["out_root_state"]) and torch.equal(out["dof_state"][..., 0], e["out_dof_pos"])
        assert (out["dof_state"][out["fall"] == 1, :, 1] == 0).all()
        available, assignment, counter, body, dof = out["available"], out["assignment"], out["counter"], out["body_state"], out["dof_state"]
