"""GPU tests of the keypoint-only task observation (env.obs_v: 7, PHC_FLAG_TASK_OBS_KP): the fused env step through the C ABI
against tests/golden/kp.npz (unmodified reference) and the oracle, the reset-path launch, the task and agent layers at observation
width 574, the keypoint MCP configuration and the composer without its final activation (ending_act: False)."""
import math

import pytest
import torch

from oracle import mcp_oracle as mo
from phc_b200 import _lib, ops, synthetic as syn
from tests import kp_oracle as KO
from tests.helpers import close, oracle_tables, smpl_step_config
from tests.kp_cases import CASES, case, config, getup_inputs, vr_track

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def smpl_cfg(**kw):
    base = dict(key_bodies=syn.SMPL_KEY_BODIES, reset_bodies=syn.SMPL_RESET_BODIES, dof_subset=syn.SMPL_DOF_SUBSET)
    base.update(kw)
    return ops.EnvStepConfig(**base)


def pack(m: syn.MotionData):
    d = m.to(DEV)
    return ops.pack_motion_lib(d.gts, d.grs, d.gvs, d.gavs, d.lrs, d.dvs, d.lengths, d.num_frames, d.dts, d.length_starts)


def make_plan(m, st, cfg, **kw):
    s = st.to(DEV)
    return ops.EnvStepPlan(cfg, pack(m), s.body_state, s.dof_state, s.dof_force, s.progress, s.motion_ids, s.start_times,
                           s.start_offsets, s.global_offset, amp_obs_buf=s.amp_hist.clone(), **{"with_ref_buffers": True, **kw})


def check(plan, exp, tag, ref_buffers=True):
    # obs atol 2e-6 as in test_gpu_env_step.py: velocity differences of O(10) operands keep one operand ulp
    close(plan.obs.cpu(), exp["obs"], atol=2e-6, what=f"{tag} obs")
    for k in ("rew", "reward_raw", "reset", "terminate", "amp_obs_buf"):
        close(getattr(plan, k).cpu(), exp[k], what=f"{tag} {k}")
    if ref_buffers:
        for k in ("ref_body_pos", "ref_body_rot", "ref_body_vel"):
            close(getattr(plan, k).cpu(), exp[k], what=f"{tag} {k}")


@pytest.mark.parametrize("tag", list(CASES))
def test_kp_env_step_vs_reference_golden(tag):
    m, st, exp, src = case(tag)
    kw, pkw = config(tag), {}
    if tag == "vr":
        kw.update(track_bodies=vr_track(src), reset_bodies=vr_track(src), full_body_reward=False)
    if tag == "occl":
        pkw = dict(occlusion=src["G_occlusion"].to(DEV).contiguous())
    if tag == "getup":
        pg, cc, ph = (t.to(DEV) for t in getup_inputs(src))
        pkw = dict(point_goal=pg, cycle_counter=cc, cycle_phase=ph)
    plan = make_plan(m, st, smpl_cfg(**kw), **pkw)
    assert plan.obs.shape[1] == exp["obs"].shape[1]
    plan.run()
    torch.cuda.synchronize()
    check(plan, exp, tag, ref_buffers=tag != "fut")
    if tag == "fut":       # fut_tracks: the reference's ref_rb_pos[..., 0, :, :] (humanoid_im.py:857-861) gives every env env 0's first sample
        close(plan.ref_body_pos[0].cpu(), exp["ref_body_pos"][0], what="fut ref_body_pos env 0")
    if tag == "getup":
        for k in ("start_times", "start_offsets", "global_offset"):
            close(plan._keep[k].cpu(), exp[k], what=f"getup {k}")
        close(pkw["point_goal"].cpu(), exp["point_goal"], what="getup point_goal")
        assert torch.equal(pkw["cycle_counter"].cpu().long(), exp["cycle_counter"].long())


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("getup", [False, True])
def test_kp_env_step_vs_oracle_4096(seed, getup):
    n = 4096
    m = syn.make_motions(n, seed=seed, min_frames=30, max_frames=90)
    st = syn.make_env_state(m, n, seed=seed, max_progress=80, with_offset=True, blend_jitter=True)
    args = (oracle_tables(m), smpl_step_config(), st.body_state, st.dof_state, st.dof_force, st.progress, st.motion_ids,
            st.start_times, st.start_offsets, st.global_offset, st.amp_hist)
    if not getup:
        plan = make_plan(m, st, smpl_cfg(obs_v=7))
        exp = KO.env_step_kp(*args)
    else:
        g = torch.Generator().manual_seed(seed)
        st.global_offset[: n // 4, :2] += torch.randn(n // 4, 2, generator=g) * 3.0       # beyond close / far distance
        pg, ph = torch.rand(n, generator=g) * 6, torch.rand(n, generator=g)
        cc = torch.randint(0, 4, (n,), generator=g, dtype=torch.int32)
        exp = KO.env_step_getup_kp(*args, pg, cc, ph, max_episode_length=60)
        pgd, ccd = pg.to(DEV), cc.to(DEV)
        plan = make_plan(m, st, smpl_cfg(obs_v=7, zero_out_far=True, cycle_motion=True, max_episode_length=60), point_goal=pgd,
                         cycle_counter=ccd, cycle_phase=ph.to(DEV))
    plan.run()
    torch.cuda.synchronize()
    assert plan.obs.shape[1] == 574
    tag = f"seed {seed} getup {getup}"
    # At 4096 random envs single columns of the unchanged v6 parts cancel larger operands than the goldens do: self-observation
    # angular velocities of O(10) (one fp32 ulp at 8..16 is 9.5e-7, rotated: up to 2.3e-6 seen) and the point-goal reward
    # 9 * (point_goal - distance) with point_goal up to 6 (9 ulps of 4..8 = 4.3e-6).  The keypoint columns keep atol 2e-6.
    close(plan.obs[:, 358:].cpu(), exp["obs"][:, 358:], atol=2e-6, what=f"{tag} task obs")
    close(plan.obs.cpu(), exp["obs"], atol=5e-6, what=f"{tag} obs")
    close(plan.rew.cpu(), exp["rew"], atol=1e-5 if getup else 1e-6, what=f"{tag} rew")
    for k in ("reward_raw", "reset", "terminate", "amp_obs_buf", "ref_body_pos", "ref_body_rot", "ref_body_vel"):
        close(getattr(plan, k).cpu(), exp[k], atol=1e-5 if (getup and k == "reward_raw") else 1e-6, what=f"{tag} {k}")
    if getup:
        close(pgd.cpu(), exp["point_goal"], what="point_goal")
        assert torch.equal(ccd.cpu(), exp["cycle_counter"].to(torch.int32))
    assert exp["reset"].sum() > 0


def test_kp_obs_only_reset_rows_equal_the_full_launch():
    n = 1000
    m = syn.make_motions(n, seed=3, min_frames=30, max_frames=90)
    st = syn.make_env_state(m, n, seed=3, max_progress=80, with_offset=True, blend_jitter=True)
    cfg = smpl_cfg(obs_v=7)
    full = make_plan(m, st, cfg)
    full.run()
    mask = torch.zeros(n, dtype=torch.int64, device=DEV)
    mask[1::3] = 1
    only = make_plan(m, st, cfg, obs=torch.full_like(full.obs, 7.0), only_where=mask, obs_only=True, with_amp=False)
    only.run()
    torch.cuda.synchronize()
    sel = mask.bool()
    assert torch.equal(only.obs[sel], full.obs[sel]) and bool((only.obs[~sel] == 7.0).all())


def _task(n, obs_v, **env):
    from phc_b200.env.humanoid_im import HumanoidIm
    return HumanoidIm({"env": {"num_envs": n, "obs_v": obs_v, **env}, "motion_data": syn.make_motions(n, seed=2), "seed": 0})


def test_humanoid_im_obs_v7_shapes_and_the_specialised_launch():
    lib = _lib.load()
    kp = _task(256, 7)
    assert kp.obs_buf.shape == (256, 574) and kp.get_task_obs_size() == 216
    d = kp.get_task_obs_size_detail()
    assert d["obs_v"] == 7 and d["target"] == 216 and len(d["track_bodies"]) == 24
    kp.reset()
    f0 = lib.phc_env_step_fast_launches()
    kp.step(None)
    torch.cuda.synchronize()
    assert lib.phc_env_step_fast_launches() == f0, "a keypoint step took a v6 specialisation"
    assert torch.isfinite(kp.obs_buf).all()
    v6 = _task(256, 6)
    assert v6.obs_buf.shape == (256, 934)
    v6.reset()
    v6.step(None)
    torch.cuda.synchronize()
    assert lib.phc_env_step_fast_launches() == f0 + 1, "the v6 steady-state launch no longer takes the specialised kernel"


@pytest.mark.parametrize("obs_v", [1, 5, 8])
def test_humanoid_im_refuses_unbuilt_observation_versions(obs_v):
    with pytest.raises(NotImplementedError, match=f"obs_v {obs_v}"):
        _task(8, obs_v)


def _agent_snapshot(n):
    from phc_b200.env.humanoid_im import HumanoidIm, RLGPUEnv
    from phc_b200.learning.amp_agent import AMPAgent
    torch.manual_seed(0)
    task = HumanoidIm({"env": {"num_envs": n, "obs_v": 7}, "motion_data": syn.make_motions(n, seed=0), "seed": 0})
    network = {"mlp": {"units": [1024, 512], "activation": "relu"}, "disc": {"units": [1024, 512], "activation": "relu"}}   # im.yaml
    agent = AMPAgent("kp", {"vec_env": RLGPUEnv(task), "seed": 0, "network": network})
    assert agent.obs_dim == 574 and agent.obs_pad == 576
    agent.obs = agent.env_reset()
    agent._init_amp_demo_buf()
    agent.train_epoch()
    torch.cuda.synchronize()
    snap = {"params": agent.model.params.clone(), "exp_avg": agent.exp_avg.clone(), "exp_avg_sq": agent.exp_avg_sq.clone(),
            "obs_mean": agent.running_mean_std.running_mean.clone()}
    losses = agent.train_result_dict()
    del agent, task
    torch.cuda.empty_cache()
    return snap, losses


def test_amp_agent_epoch_at_obs_width_574_is_finite_and_reproducible():
    a, la = _agent_snapshot(4096)
    b, lb = _agent_snapshot(4096)
    assert la and all(math.isfinite(v) for v in la.values()), la
    assert all(torch.isfinite(v).all() for v in a.values())
    differ = [k for k in a if not torch.equal(a[k], b[k])]
    assert not differ, f"state differs between two identically seeded runs: {differ}"
    assert la == lb


def _pnn_checkpoint(obs_dim, act_dim, K, units=(64, 32), seed=0):
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


def test_humanoid_im_mcp_with_a_keypoint_pnn():
    """phc_kp_mcp_iccv-style task: keypoint observation (574 columns) into primitives whose first layer is [units, 574]."""
    from phc_b200.env.humanoid_im_mcp import HumanoidImMCP
    n, K = 64, 3
    m = syn.make_motions(n, seed=4, min_frames=40, max_frames=90)
    ck = _pnn_checkpoint(574, 69, K)
    task = HumanoidImMCP({"env": {"num_envs": n, "obs_v": 7, "num_prim": K, "has_pnn": True, "has_lateral": False}, "motion_data": m,
                          "seed": 4}, pnn_checkpoint=ck)
    assert task.get_obs_size() == 574 and task.get_action_size() == K
    task.reset()
    w = torch.relu(torch.randn(n, K, generator=torch.Generator().manual_seed(1))).to(DEV)
    got = task.compose_actions(w).clone()
    torch.cuda.synchronize()
    exp = mo.mcp_step_actions(task.obs_buf.cpu(), ck["running_mean_std"]["running_mean"], ck["running_mean_std"]["running_var"], ck["model"],
                              w.cpu(), K, dtype=torch.float64)
    err = (got.cpu().double() - exp).abs().max().item()
    assert err <= 1e-5 * max(exp.abs().max().item(), 1e-3), err
    task.step(w)
    torch.cuda.synchronize()
    assert torch.isfinite(task.obs_buf).all()


@pytest.mark.parametrize("activation", ["relu", "silu"])
def test_composer_without_ending_activation_forward_backward(activation):
    """network.ending_act: False (phc_comp_kp_2 on im_mcp_big): the composer's last Linear has no activation after it
    (amp_network_mcp_builder.py:58-59).  Forward and weight / bias gradients against autograd in fp64."""
    from phc_b200.learning.networks import AMPNetwork, MLPEngine, round4
    D, K, units, B = 574, 4, [256, 128], 512
    net = AMPNetwork(D, K, 8, units=units, disc_units=(8,), activation=activation, device=DEV, kind="amp_mcp", num_prim=K, ending_act=False)
    assert not net.actor.head_relu
    sd = {k: v.detach().cpu() for k, v in net.state_dict().items() if ".composer." in k}
    eng = MLPEngine(net)
    x_ref = torch.randn(B, D, generator=torch.Generator().manual_seed(3))
    x = torch.zeros(B, round4(D), device=DEV)
    x[:, :D] = x_ref.to(DEV)
    ws = eng.workspace("a", net.actor, B)
    out = eng.forward(net.actor, x, ws)[:, :K].clone()
    c64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    ref = mo.mlp_forward(c64, "a2c_network.composer.", x_ref.double(), ending_act=False, act=activation)
    assert bool((ref < 0).any()), "a linear head reaches negative values"
    _close_scale(out, ref.detach(), "composer forward", 1e-5)
    dout = torch.randn(B, K, generator=torch.Generator().manual_seed(6))
    ws["dout"].zero_()
    ws["dout"][:, :K] = dout.to(DEV)
    net.grads.zero_()
    eng.backward(net.actor, x, ws)
    torch.cuda.synchronize()
    (ref * dout.double()).sum().backward()
    for l in net.actor.layers:
        _close_scale(net.weight(l, True)[:, :l.in_dim], c64[f"a2c_network.{l.name}.weight"].grad, f"{l.name}.weight grad", 2e-5)
        _close_scale(net.bias(l, True), c64[f"a2c_network.{l.name}.bias"].grad, f"{l.name}.bias grad", 2e-5)


def _close_scale(got, ref, what, tol):
    ref = ref.to(torch.float64)
    err = (got.detach().cpu().to(torch.float64) - ref).abs().max().item()
    scale = max(ref.abs().max().item(), 1e-3)
    assert err <= tol * scale, f"{what}: max err {err:.3e} > {tol:g} * {scale:.3e}"
