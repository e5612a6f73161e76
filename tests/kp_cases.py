"""The cases of tests/golden/kp.npz (make_golden_kp.py): the keypoint-only observation (env.obs_v: 7) of the unmodified reference on
the inputs of existing goldens.  Shared by the oracle, emulation and GPU tests (test infrastructure)."""
import torch

from phc_b200 import synthetic as syn
from tests.helpers import load, motion_data_from

# case -> (source golden, prefix of its input arrays, prefix of its outputs for the same inputs: the AMP observation, which obs_v
# does not change, is compared against these)
CASES = {"A": ("envstep.npz", "A_in_", "A_out_"), "B": ("envstep.npz", "B_in_", "B_out_"), "C": ("envstep.npz", "A_in_", "C_out_"),
         "fut": ("fut.npz", "in_", "out_"), "getup": ("getup.npz", "in_", "out_"), "occl": ("vr.npz", "in_", "G_out_"),
         "vr": ("vr.npz", "in_", "E_out_")}
KEYS = ("obs", "rew", "reward_raw", "reset", "terminate", "ref_body_pos", "ref_body_rot", "ref_body_vel")


def case(tag):
    """(motion data, env state, expected outputs, extra source arrays) of one case; expected includes amp_obs_buf."""
    name, pin, pout = CASES[tag]
    src, kp = load(name), load("kp.npz")
    m = motion_data_from(src)
    st = syn.EnvState(**{k: src[pin + k].clone() for k in syn.EnvState.__dataclass_fields__})
    exp = {k[len(tag) + 5:]: v for k, v in kp.items() if k.startswith(f"{tag}_out_")}
    exp["amp_obs_buf"] = src[pout + "amp_obs_buf"]
    return m, st, exp, src


def config(tag):
    """ops.EnvStepConfig / oracle StepConfig keyword arguments of a case (besides the SMPL defaults)."""
    kw = dict(obs_v=7)
    if tag == "C":
        kw.update(upright=False, local_root_obs=False)
    if tag == "fut":
        kw.update(time_steps=3, traj_dt=1 / 10)
    if tag == "getup":
        kw.update(zero_out_far=True, cycle_motion=True, max_episode_length=15)
    return kw


def vr_track(src):
    return src["track"].tolist()


def getup_inputs(src):
    return src["in_point_goal"].clone(), src["in_cycle_counter"].to(torch.int32).clone(), src["in_cycle_phase"].clone()
