"""The fused env-step KERNEL SOURCE on the CPU: phc_b200/csrc/env_step.cu (kernel + layout helpers, verbatim), phc_math.cuh and
the reductions of phc_common.cuh are compiled with g++ against a small emulation of the CUDA constructs they use
(tests/emu/: one warp = 32 threads, barrier-based warp collectives, mbarrier / TMA bulk copy stand-ins) and run on the goldens
of the UNMODIFIED reference -- the same comparisons tests/test_gpu_env_step.py / test_gpu_getup.py make on the GPU, here without
a GPU.  The arguments are assembled by the product's own ops.EnvStepPlan (on host tensors).  Tolerances as on the GPU."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

from phc_b200 import _lib, ops, synthetic as syn          # noqa: E402
from tests.helpers import close, env_state_from, load, motion_data_from   # noqa: E402


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    import shutil
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    import build_emu
    import host_plan
    return host_plan.Emu(build_emu.build(str(tmp_path_factory.mktemp("emu")))), host_plan


def smpl_cfg(**kw):
    base = dict(key_bodies=syn.SMPL_KEY_BODIES, reset_bodies=syn.SMPL_RESET_BODIES, dof_subset=syn.SMPL_DOF_SUBSET)
    base.update(kw)
    return ops.EnvStepConfig(**base)


def make_plan(hp, m, st, cfg, **kw):
    mlib = hp.host_pack(m.gts, m.grs, m.gvs, m.gavs, m.lengths, m.num_frames, m.dts, m.length_starts)
    s = st
    with hp.host_mode():
        return ops.EnvStepPlan(cfg, mlib, s.body_state.clone(), s.dof_state.clone(), s.dof_force.clone(), s.progress.clone(), s.motion_ids.clone(),
                               s.start_times.clone(), s.start_offsets.clone(), s.global_offset.clone(), amp_obs_buf=s.amp_hist.clone(),
                               with_ref_buffers=kw.pop("with_ref_buffers", True), **kw)


def check(plan, exp, tag, ref_buffers=True):
    close(plan.obs, exp["obs"], atol=2e-6, what=f"{tag} obs")
    close(plan.rew, exp["rew"], what=f"{tag} rew")
    close(plan.reward_raw, exp["reward_raw"], what=f"{tag} reward_raw")
    close(plan.reset, exp["reset"], what=f"{tag} reset")
    close(plan.terminate, exp["terminate"], what=f"{tag} terminate")
    close(plan.amp_obs_buf, exp["amp_obs_buf"], what=f"{tag} amp_obs_buf")
    if ref_buffers:
        for k in ("ref_body_pos", "ref_body_rot", "ref_body_vel"):
            close(getattr(plan, k), exp[k], what=f"{tag} {k}")


@pytest.mark.parametrize("tag,in_tag,kw", [("A", "A", {}), ("B", "B", {}), ("C", "A", dict(upright=False, local_root_obs=False)),
                                            ("D", "B", dict(term_use_mean=True))])
def test_kernel_source_vs_reference_golden(emu, tag, in_tag, kw):
    e, hp = emu
    g = load("envstep.npz")
    plan = make_plan(hp, motion_data_from(g), env_state_from(g, in_tag), smpl_cfg(**kw))
    e.run(plan, "smpl")
    check(plan, {k: g[f"{tag}_out_{k}"] for k in ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf", "ref_body_pos", "ref_body_rot", "ref_body_vel")}, tag)


@pytest.mark.parametrize("tag", ["E", "F", "G"])
def test_tracked_subset_occlusion_and_shape_columns(emu, tag):
    """vr.npz (make_golden.gen_vr, the unmodified reference): env_vr.yaml's Head + hands subset with the subset reward and the shape /
    limb-weight columns (E), the subset with the full-body reward (F), occlusion training (G) -- through the generic instantiation."""
    e, hp = emu
    g = load("vr.npz")
    track = g["track"].tolist()
    subset = tag in ("E", "F")
    cfg = smpl_cfg(track_bodies=track if subset else None, reset_bodies=track if subset else syn.SMPL_RESET_BODIES, full_body_reward=tag != "E")
    st = syn.EnvState(**{k: g[f"in_{k}"] for k in syn.EnvState.__dataclass_fields__})
    kw = {}
    if tag == "E":
        kw = dict(shape_params=g["E_shape"][:, :-6].contiguous(), limb_weights=g["E_limb"].contiguous())
    if tag == "G":
        kw = dict(occlusion=g["G_occlusion"].contiguous())
    plan = make_plan(hp, motion_data_from(g), st, cfg, **kw)
    assert plan.obs.shape[1] == g[f"{tag}_out_obs"].shape[1]
    e.run(plan, "generic")
    check(plan, {k: g[f"{tag}_out_{k}"] for k in ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf", "ref_body_pos", "ref_body_rot", "ref_body_vel")}, tag)


def test_generic_instantiation_matches_too(emu):
    e, hp = emu
    g = load("envstep.npz")
    plan = make_plan(hp, motion_data_from(g), env_state_from(g, "B"), smpl_cfg())
    e.run(plan, "generic")
    check(plan, {k: g[f"B_out_{k}"] for k in ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf", "ref_body_pos", "ref_body_rot", "ref_body_vel")}, "B generic")


def test_future_tracks_instantiation(emu):
    e, hp = emu
    g = load("fut.npz")
    st = syn.EnvState(**{k: g[f"in_{k}"] for k in syn.EnvState.__dataclass_fields__})
    plan = make_plan(hp, motion_data_from(g), st, smpl_cfg(time_steps=3, traj_dt=1 / 10))
    e.run(plan, "fut")
    check(plan, {k: g[f"out_{k}"] for k in ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf")}, "fut", ref_buffers=False)
    close(plan.ref_body_pos[0], g["out_ref_body_pos"][0], what="fut ref_body_pos env 0")


def test_getup_instantiation_vs_reference_golden(emu):
    e, hp = emu
    g = load("getup.npz")
    st = syn.EnvState(**{k: g[f"in_{k}"] for k in syn.EnvState.__dataclass_fields__})
    pg, cc, ph = g["in_point_goal"].clone(), g["in_cycle_counter"].to(torch.int32).clone(), g["in_cycle_phase"].clone()
    plan = make_plan(hp, motion_data_from(g), st, smpl_cfg(zero_out_far=True, cycle_motion=True, max_episode_length=15), point_goal=pg,
                     cycle_counter=cc, cycle_phase=ph)
    e.run(plan, "getup")
    exp = {k[4:]: v for k, v in g.items() if k.startswith("out_")}
    check(plan, exp, "getup")
    k = plan._keep
    close(k["start_times"], exp["start_times"], what="getup start_times")
    close(k["start_offsets"], exp["start_offsets"], what="getup start_offsets")
    close(k["global_offset"], exp["global_offset"], what="getup global_offset")
    close(pg, exp["point_goal"], what="getup point_goal")
    assert torch.equal(cc.long(), exp["cycle_counter"].long())


@pytest.mark.parametrize("frames", [(30, 50), (4, 12)])
def test_specialised_instantiation_and_pose_cache(emu, frames):
    """(The second parametrisation uses clips of 4-12 frames with progress up to 20: most envs are past the end of their clip, where
    the bracket collapses onto the last frame -- one copy for both slots -- and pass_time resets fire.)
    Two consecutive steps through the pose cache: step 1 (generic, fills the cache with the pose interpolated for its
    observation), step 2 through the FAST instantiation (reward pose from the cache, ring slot, bulk rows) against the generic
    instantiation without cache on the same inputs -- the arithmetic is the same source, so the results agree to rounding."""
    e, hp = emu
    n = 12
    m = syn.make_motions(n, seed=5, min_frames=frames[0], max_frames=frames[1])
    st = syn.make_env_state(m, n, seed=5, max_progress=20)
    bs = hp.round4(13 * 24)
    cache = torch.zeros(n, bs)
    warm = make_plan(hp, m, st, smpl_cfg(), with_ref_buffers=False, ref_cache=cache)
    e.run(warm, "smpl")                                         # cache := pose at (progress + 1) dt
    st2 = syn.EnvState(**{**{k: getattr(st, k) for k in st.__dataclass_fields__}, "progress": st.progress + 1})
    ref_plan = make_plan(hp, m, st2, smpl_cfg())
    e.run(ref_plan, "smpl")
    fast = make_plan(hp, m, st2, smpl_cfg(), with_ref_buffers=False, ref_cache=cache.clone(), reward_from_cache=True, amp_ring=True)
    fast.advance_ring()
    assert fast.args.flags == e.lib.emu_fast_flags()
    e.run(fast, "fast")
    close(fast.obs, ref_plan.obs, atol=2e-6, what="fast obs")
    close(fast.rew, ref_plan.rew, what="fast rew")
    close(fast.reward_raw, ref_plan.reward_raw, what="fast reward_raw")
    assert torch.equal(fast.reset, ref_plan.reset) and torch.equal(fast.terminate, ref_plan.terminate)
    close(fast.amp_obs_buf[:, fast.ring_head], ref_plan.amp_obs_buf[:, 0], what="fast AMP ring slot")
    close(fast.ref_cache[:, :13 * 24].view(n, 24, 13)[..., 0:3], ref_plan.ref_body_pos, what="fast pose cache")
    assert float(fast.obs_full_row_pad_max if hasattr(fast, "obs_full_row_pad_max") else 0.0) == 0.0
    # env_step_fast.cu (what phc_env_step launches for this configuration: the same arithmetic and reductions, phases ordered by
    # input arrival, the observation row staged in two pieces) against the FAST instantiation: every output bit for bit
    fk = make_plan(hp, m, st2, smpl_cfg(), with_ref_buffers=False, ref_cache=cache.clone(), reward_from_cache=True, amp_ring=True)
    fk.advance_ring()
    e.run(fk, "fastk")
    for k in ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf", "ref_cache"):
        assert torch.equal(getattr(fk, k), getattr(fast, k)), f"env_step_fast_kernel {k}"


# ---- env_step_wide.cu: the strided kernel for more than 32 bodies (and, as a cross-check, for the 24-body goldens) ----------
@pytest.mark.parametrize("tag,in_tag,kw", [("A", "A", {}), ("B", "B", {}), ("C", "A", dict(upright=False, local_root_obs=False)),
                                            ("D", "B", dict(term_use_mean=True))])
def test_wide_kernel_on_the_24_body_goldens(emu, tag, in_tag, kw):
    e, hp = emu
    g = load("envstep.npz")
    plan = make_plan(hp, motion_data_from(g), env_state_from(g, in_tag), smpl_cfg(**kw))
    e.run(plan, "wide")
    check(plan, {k: g[f"{tag}_out_{k}"] for k in ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf", "ref_body_pos", "ref_body_rot", "ref_body_vel")}, f"wide {tag}")


def test_wide_kernel_smplx_52_bodies_vs_reference_golden(emu):
    e, hp = emu
    g = load("smplx.npz")
    st = syn.EnvState(**{k: g[f"in_{k}"] for k in syn.EnvState.__dataclass_fields__})
    cfg = ops.EnvStepConfig(key_bodies=syn.SMPLX_KEY_BODIES, reset_bodies=None, dof_subset=None)
    plan = make_plan(hp, motion_data_from(g), st, cfg)
    assert plan.obs.shape[1] == 1 + 15 * 52 - 3 + 24 * 52
    e.run(plan, "wide")
    check(plan, {k: g[f"out_{k}"] for k in ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf", "ref_body_pos", "ref_body_rot", "ref_body_vel")}, "smplx")


def test_wide_kernel_g1_39_bodies_vs_reference_golden(emu):
    e, hp = emu
    g = load("g1.npz")
    f = lambda k: g["tab_" + k]
    cfg = ops.EnvStepConfig(key_bodies=syn.G1_KEY_BODIES, reset_bodies=None, dof_subset=None, ext_parents=syn.G1_EXT_PARENTS, ext_pos=syn.G1_EXT_POS)
    for tag in ("A", "B"):
        st = syn.EnvState(**{k: g[f"{tag}_in_{k}"] for k in syn.EnvState.__dataclass_fields__})
        mlib = hp.host_pack(f("gts_t"), f("grs_t"), f("gvs_t"), f("gavs_t"), f("lengths"), f("num_frames"), f("dts"), f("length_starts"),
                            num_ext=1, num_dofs=syn.G1_NUM_DOFS)
        with hp.host_mode():
            plan = ops.EnvStepPlan(cfg, mlib, st.body_state.clone(), st.dof_state.clone(), st.dof_force.clone(), st.progress.clone(),
                                   st.motion_ids.clone(), st.start_times.clone(), st.start_offsets.clone(), st.global_offset.clone(),
                                   amp_obs_buf=st.amp_hist.clone(), with_ref_buffers=True)
        assert plan.obs.shape[1] == 1 + 15 * 38 - 3 + 24 * 38 and plan.amp_dim == 13 + 2 * 37 + 12
        e.run(plan, "wide")
        check(plan, {k: g[f"{tag}_out_{k}"] for k in ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf", "ref_body_pos", "ref_body_rot", "ref_body_vel")}, f"g1 {tag}")


def test_wide_kernel_pose_cache_and_obs_only(emu):
    """Pose cache through the wide kernel (step 1 fills it, step 2 reads the reward pose from it) and the masked observation-only
    launch of the reset path, against the same kernel without cache / mask."""
    e, hp = emu
    g = load("smplx.npz")
    st = syn.EnvState(**{k: g[f"in_{k}"] for k in syn.EnvState.__dataclass_fields__})
    m = motion_data_from(g)
    n, J = st.body_state.shape[0], 52
    cfg = ops.EnvStepConfig(key_bodies=syn.SMPLX_KEY_BODIES, reset_bodies=None, dof_subset=None)
    cache = torch.zeros(n, hp.round4(13 * J))
    e.run(make_plan(hp, m, st, cfg, with_ref_buffers=False, ref_cache=cache), "wide")
    st2 = syn.EnvState(**{**{k: getattr(st, k) for k in st.__dataclass_fields__}, "progress": st.progress + 1})
    plain = make_plan(hp, m, st2, cfg)
    e.run(plain, "wide")
    cached = make_plan(hp, m, st2, cfg, with_ref_buffers=False, ref_cache=cache, reward_from_cache=True)
    e.run(cached, "wide")
    for k in ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf"):
        assert torch.equal(getattr(cached, k), getattr(plain, k)), k            # same source, same operands: bit-identical
    mask = torch.zeros(n, dtype=torch.int64)
    mask[1::3] = 1
    only = make_plan(hp, m, st2, cfg, obs=torch.full_like(plain.obs, 7.0).contiguous(), only_where=mask, obs_only=True, with_amp=False)
    e.run(only, "wide")
    assert torch.equal(only.obs[mask.bool()], plain.obs[mask.bool()]) and bool((only.obs[~mask.bool()] == 7.0).all())


def test_wide_kernel_getup_smplx_vs_reference_golden(emu):
    """env_im_x_getup_mcp.yaml: zero_out_far + cycle_motion at 52 bodies through the strided kernel."""
    e, hp = emu
    g = load("getup_smplx.npz")
    st = syn.EnvState(**{k: g[f"in_{k}"] for k in syn.EnvState.__dataclass_fields__})
    pg, cc, ph = g["in_point_goal"].clone(), g["in_cycle_counter"].to(torch.int32).clone(), g["in_cycle_phase"].clone()
    cfg = ops.EnvStepConfig(key_bodies=syn.SMPLX_KEY_BODIES, reset_bodies=None, dof_subset=None, zero_out_far=True, cycle_motion=True, max_episode_length=15)
    plan = make_plan(hp, motion_data_from(g), st, cfg, point_goal=pg, cycle_counter=cc, cycle_phase=ph)
    e.run(plan, "wide")
    exp = {k[4:]: v for k, v in g.items() if k.startswith("out_")}
    check(plan, exp, "getup smplx")
    k = plan._keep
    close(k["start_times"], exp["start_times"], what="start_times")
    close(k["start_offsets"], exp["start_offsets"], what="start_offsets")
    close(k["global_offset"], exp["global_offset"], what="global_offset")
    close(pg, exp["point_goal"], what="point_goal")
    assert torch.equal(cc.long(), exp["cycle_counter"].long())


def test_wide_kernel_getup_on_the_24_body_golden(emu):
    e, hp = emu
    g = load("getup.npz")
    st = syn.EnvState(**{k: g[f"in_{k}"] for k in syn.EnvState.__dataclass_fields__})
    pg, cc, ph = g["in_point_goal"].clone(), g["in_cycle_counter"].to(torch.int32).clone(), g["in_cycle_phase"].clone()
    plan = make_plan(hp, motion_data_from(g), st, smpl_cfg(zero_out_far=True, cycle_motion=True, max_episode_length=15), point_goal=pg,
                     cycle_counter=cc, cycle_phase=ph)
    e.run(plan, "wide")
    exp = {k[4:]: v for k, v in g.items() if k.startswith("out_")}
    check(plan, exp, "getup (wide kernel)")
    close(plan._keep["global_offset"], exp["global_offset"], what="global_offset")
    assert torch.equal(cc.long(), exp["cycle_counter"].long())


def test_chaos_mode_subset():
    """The same emulation with every lane dawdling randomly after each collective (PHC_EMU_CHAOS=1, read when the emulation
    library loads, hence a fresh process): lanes drift as far apart as the synchronisation allows, so a missing __syncwarp()
    turns into a wrong result.  Runs the cases with the most cross-lane traffic."""
    import subprocess
    if os.environ.get("PHC_EMU_CHAOS") == "1":
        pytest.skip("already inside the chaos run")
    env = dict(os.environ, PHC_EMU_CHAOS="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-p", "no:cacheprovider", "-k",
                        "getup or specialised or wide_kernel_on_the_24_body_goldens or golden[B"], capture_output=True, text=True, env=env,
                       cwd=os.path.dirname(HERE), timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


def test_wide_kernel_future_tracks_and_eval_extras(emu):
    """The strided kernel on fut.npz (T = 3) and its im_eval extras (mpjpe, body_pos_gt) against the oracle."""
    from oracle import phc_oracle as O
    from tests.helpers import smpl_step_config, tables_from
    e, hp = emu
    g = load("fut.npz")
    st = syn.EnvState(**{k: g[f"in_{k}"] for k in syn.EnvState.__dataclass_fields__})
    plan = make_plan(hp, motion_data_from(g), st, smpl_cfg(time_steps=3, traj_dt=1 / 10), with_eval_extras=True)
    e.run(plan, "wide")
    check(plan, {k: g[f"out_{k}"] for k in ("obs", "rew", "reward_raw", "reset", "terminate", "amp_obs_buf")}, "wide fut", ref_buffers=False)
    exp = O.env_step(tables_from(g), smpl_step_config(time_steps=3, traj_dt=1 / 10), st.body_state, st.dof_state, st.dof_force, st.progress,
                     st.motion_ids, st.start_times, st.start_offsets, st.global_offset, st.amp_hist)
    close(plan.mpjpe, exp["mpjpe"], what="mpjpe")
    close(plan.body_pos_gt, exp["body_pos_gt"], what="body_pos_gt")
    for k in ("ref_body_pos", "ref_body_rot", "ref_body_vel"):
        close(getattr(plan, k), exp[k], what=k)
    # and the staged kernel's extras on the same inputs
    plan2 = make_plan(hp, motion_data_from(g), st, smpl_cfg(time_steps=3, traj_dt=1 / 10), with_eval_extras=True)
    e.run(plan2, "fut")
    close(plan2.mpjpe, exp["mpjpe"], what="mpjpe (staged kernel)")
    close(plan2.body_pos_gt, exp["body_pos_gt"], what="body_pos_gt (staged kernel)")
