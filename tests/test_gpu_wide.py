"""GPU parity of the strided kernels for more than 32 bodies (env_step_wide.cu, motion_wide.cu): Unitree G1 (38 + 1 bodies, 37
hinge dofs) and SMPL-X (52 bodies) against the goldens of the unmodified reference.

The CPU emulation of the same kernel sources
(tests/test_env_step_emu_cpu.py, tests/test_motion_emu_cpu.py) checks them against the same goldens without a GPU."""
import os

import pytest
import torch

from phc_b200 import ops, synthetic as syn
from tests.helpers import close, load, motion_data_from
from tests.test_gpu_env_step import check_against, run_cuda_step

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEYS = ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf", "ref_body_pos", "ref_body_rot", "ref_body_vel")


def test_smplx_env_step_vs_reference_golden():
    g = load("smplx.npz")
    st = syn.EnvState(**{k: g[f"in_{k}"] for k in syn.EnvState.__dataclass_fields__})
    cfg = ops.EnvStepConfig(key_bodies=syn.SMPLX_KEY_BODIES, reset_bodies=None, dof_subset=None)
    plan = run_cuda_step(motion_data_from(g), st, cfg)
    check_against(plan, {k: g[f"out_{k}"] for k in KEYS}, "smplx")


def _g1_lib(g):
    f = lambda k: g["tab_" + k].to(DEV)
    return ops.pack_robot_motion_lib(f("gts_t"), f("grs_t"), f("gvs_t"), f("gavs_t"), f("dof_pos"), f("dvs"), syn.G1_NUM_BODIES, f("lengths"),
                                     f("num_frames"), f("dts"), f("length_starts"))


def test_g1_env_step_motion_state_and_demo_vs_reference_golden():
    g = load("g1.npz")
    mlib = _g1_lib(g)
    res = ops.motion_state(mlib, g["ms_ids"].to(DEV), g["ms_times"].to(DEV), g["ms_offset"].to(DEV))
    for k in ("root_pos", "root_rot", "dof_pos", "root_vel", "root_ang_vel", "dof_vel", "rg_pos", "rb_rot", "body_vel", "body_ang_vel",
              "rg_pos_t", "rg_rot_t", "body_vel_t", "body_ang_vel_t"):
        close(res[k].cpu(), g["ms_out_" + k], what="g1 motion_state " + k)
    cfg = ops.EnvStepConfig(key_bodies=syn.G1_KEY_BODIES, reset_bodies=None, dof_subset=None, ext_parents=syn.G1_EXT_PARENTS, ext_pos=syn.G1_EXT_POS)
    for tag in ("A", "B"):
        st = syn.EnvState(**{k: g[f"{tag}_in_{k}"] for k in syn.EnvState.__dataclass_fields__}).to(DEV)
        plan = ops.EnvStepPlan(cfg, mlib, st.body_state, st.dof_state, st.dof_force, st.progress, st.motion_ids, st.start_times, st.start_offsets,
                               st.global_offset, amp_obs_buf=st.amp_hist.clone(), with_ref_buffers=True)
        plan.run()
        torch.cuda.synchronize()
        check_against(plan, {k: g[f"{tag}_out_{k}"] for k in KEYS}, f"g1 {tag}")
    demo = ops.amp_obs_demo(mlib, cfg, g["demo_ids"].to(DEV), g["demo_t0"].to(DEV))
    close(demo.cpu(), g["demo_out"], rtol=1e-4, atol=2e-5, what="g1 amp_obs_demo")


def test_smplx_getup_vs_reference_golden():
    """env_im_x_getup_mcp.yaml: zero_out_far + cycle_motion at 52 bodies."""
    g = load("getup_smplx.npz")
    st = syn.EnvState(**{k: g[f"in_{k}"] for k in syn.EnvState.__dataclass_fields__}).to(DEV)
    from tests.test_gpu_env_step import pack
    mlib = pack(motion_data_from(g))
    pg, cc, ph = g["in_point_goal"].to(DEV).clone(), g["in_cycle_counter"].to(DEV).to(torch.int32).clone(), g["in_cycle_phase"].to(DEV).clone()
    cfg = ops.EnvStepConfig(key_bodies=syn.SMPLX_KEY_BODIES, reset_bodies=None, dof_subset=None, zero_out_far=True, cycle_motion=True, max_episode_length=15)
    plan = ops.EnvStepPlan(cfg, mlib, st.body_state, st.dof_state, st.dof_force, st.progress, st.motion_ids, st.start_times, st.start_offsets,
                           st.global_offset, amp_obs_buf=st.amp_hist.clone(), with_ref_buffers=True, point_goal=pg, cycle_counter=cc, cycle_phase=ph)
    plan.run()
    torch.cuda.synchronize()
    exp = {k[4:]: v for k, v in g.items() if k.startswith("out_")}
    check_against(plan, exp, "getup smplx")
    close(st.global_offset.cpu(), exp["global_offset"], what="global_offset")
    close(pg.cpu(), exp["point_goal"], what="point_goal")
    assert torch.equal(cc.cpu().long(), exp["cycle_counter"].long())


def test_g1_task_rollout_and_agent_epoch():
    """HumanoidIm with Unitree G1 shaped robot tables (38 bodies + 1 extend body, 37 hinge dofs): reset / step against the
    oracle, then one AMPAgent epoch -- every kernel of the path on the strided variants."""
    from oracle import phc_oracle as O
    from phc_b200.env.humanoid_im import HumanoidIm, RLGPUEnv
    from phc_b200.learning.amp_agent import AMPAgent
    n = 64
    m = syn.make_robot_motions(n, seed=8, num_bodies=syn.G1_NUM_BODIES, num_dofs=syn.G1_NUM_DOFS, ext_parents=syn.G1_EXT_PARENTS,
                               ext_pos=syn.G1_EXT_POS, min_frames=40, max_frames=90)
    ext = [dict(parent=p, pos=q) for p, q in zip(syn.G1_EXT_PARENTS, syn.G1_EXT_POS)]
    task = HumanoidIm({"env": {"num_envs": n, "key_body_ids": syn.G1_KEY_BODIES}, "motion_data": m, "seed": 8, "extend_config": ext,
                       "humanoid_type": "g1"})
    J, D = syn.G1_NUM_BODIES, syn.G1_NUM_DOFS
    assert task.get_obs_size() == 1 + 15 * J - 3 + 24 * J and task.get_action_size() == D
    task.reset()
    hist = task._amp_obs_buf.cpu().clone()
    task.step(None)
    torch.cuda.synchronize()
    tab = O.RobotTables(m.gts_t, m.grs_t, m.gvs_t, m.gavs_t, m.dof_pos, m.dvs, m.lengths, m.num_frames, m.dts, m.length_starts, J)
    cfg = O.StepConfig(key_bodies=syn.G1_KEY_BODIES, reset_bodies=None, dof_subset=None)
    exp = O.env_step_robot(tab, cfg, syn.G1_EXT_PARENTS, syn.G1_EXT_POS, task._rigid_body_state_reshaped.cpu(), task._dof_state.cpu(),
                           task.dof_force_tensor.cpu(), task.progress_buf.cpu(), task._sampled_motion_ids.cpu(), task._motion_start_times.cpu(),
                           torch.zeros(n), torch.zeros(n, 3), hist)
    close(task.obs_buf.cpu(), exp["obs"], atol=2e-6, what="task obs")
    close(task.rew_buf.cpu(), exp["rew"], what="task rew")
    close(task.reset_buf.cpu(), exp["reset"], what="task reset")
    close(task._amp_obs_buf.cpu(), exp["amp_obs_buf"], what="task amp window")
    agent = AMPAgent("t", {"vec_env": RLGPUEnv(task), "horizon_length": 8, "minibatch_size": 256, "amp_minibatch_size": 64, "mini_epochs": 2,
                           "amp_obs_demo_buffer_size": 2048, "amp_replay_buffer_size": 2048, "amp_batch_size": 128,
                           "network": {"mlp": {"units": [128, 64], "activation": "relu"}, "disc": {"units": [128, 64], "activation": "relu"}}})
    agent.obs = agent.env_reset()
    agent._init_amp_demo_buf()
    p0 = agent.model.params.clone()
    agent.train_epoch()
    torch.cuda.synchronize()
    assert torch.isfinite(agent.model.params).all() and not torch.equal(agent.model.params, p0)
