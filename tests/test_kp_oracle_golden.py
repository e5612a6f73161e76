"""The keypoint-only task observation oracle (tests/kp_oracle.py) against tests/golden/kp.npz, produced by the unmodified reference
with env.obs_v = 7.  CPU only; tolerances of test_oracle_golden.py (rtol 1e-5 / atol 1e-6)."""
import pytest
import torch

from tests import kp_oracle as KO
from tests.helpers import close, oracle_tables, smpl_step_config
from tests.kp_cases import CASES, case, getup_inputs, vr_track


def _cfg(tag, src):
    kw = {}
    if tag == "C":
        kw = dict(upright=False, local_root_obs=False)
    if tag == "fut":
        kw = dict(time_steps=3, traj_dt=1 / 10)
    if tag == "vr":
        kw = dict(track_bodies=vr_track(src), reset_bodies=vr_track(src), full_body_reward=False)
    return smpl_step_config(**kw)


@pytest.mark.parametrize("tag", list(CASES))
def test_kp_oracle_vs_reference_golden(tag):
    m, st, exp, src = case(tag)
    tab, cfg = oracle_tables(m), _cfg(tag, src)
    args = (tab, cfg, st.body_state, st.dof_state, st.dof_force, st.progress, st.motion_ids, st.start_times, st.start_offsets,
            st.global_offset, st.amp_hist)
    if tag == "getup":
        pg, cc, ph = getup_inputs(src)
        out = KO.env_step_getup_kp(*args, pg, cc, ph, max_episode_length=15)
        for k in ("start_times", "start_offsets", "global_offset", "point_goal"):
            close(out[k], exp[k], what=f"getup {k}")
        assert torch.equal(out["cycle_counter"].long(), exp["cycle_counter"].long())
    else:
        out = KO.env_step_kp(*args, occlusion=src["G_occlusion"] if tag == "occl" else None)
    J = st.body_state.shape[1]
    K = len(vr_track(src)) if tag == "vr" else J
    assert exp["obs"].shape[1] == 1 + 15 * J - 3 + 9 * K * (3 if tag == "fut" else 1)
    for k in ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf"):
        close(out[k], exp[k], what=f"{tag} {k}")
    for k in ("ref_body_pos", "ref_body_rot", "ref_body_vel"):
        if tag == "fut":       # fut_tracks: the reference's ref_rb_pos[..., 0, :, :] (humanoid_im.py:857-861) gives every env env 0's first sample
            close(out[k][0], exp[k][0], what=f"fut {k} env 0")
        else:
            close(out[k], exp[k], what=f"{tag} {k}")


def test_smpl_keypoint_observation_is_574_wide():
    _, _, exp, _ = case("A")
    assert exp["obs"].shape[1] == 358 + 216 == 574


def test_occluded_body_keeps_the_reference_velocity():
    """v7 replaces an occluded body's reference position only (humanoid_im.py:847-851): its diff_pos is zero, its diff_vel is not."""
    m, st, exp, src = case("occl")
    oc = src["G_occlusion"].bool()
    J = oc.shape[1]
    task = exp["obs"][:, 1 + 15 * J - 3:].view(-1, 3, J, 3)
    assert oc.any()
    assert torch.all(task[:, 0][oc] == 0)
    assert torch.all(task[:, 1][oc].abs().sum(-1) > 0)
