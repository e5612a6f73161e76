"""The keypoint instantiations of the fused env-step kernel (KP = true, PHC_FLAG_TASK_OBS_KP) on the CPU: the kernel source through
the emulation of tests/emu (verbatim product source, one warp = 32 threads), arguments assembled by ops.EnvStepPlan on host tensors,
against tests/golden/kp.npz from the unmodified reference.  Also the C ABI sizes and refusals of the keypoint observation, which
need no device."""
import ctypes as C
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

from phc_b200 import _lib, ops, synthetic as syn          # noqa: E402
from tests.helpers import close                           # noqa: E402
from tests.kp_cases import case, config, getup_inputs, vr_track   # noqa: E402


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    import shutil
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    import host_plan
    import kp_emu
    return kp_emu.EmuKp(kp_emu.build(str(tmp_path_factory.mktemp("emu_kp")))), host_plan


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
                               with_ref_buffers=True, **kw)


def run_case(e, hp, tag, variant):
    m, st, exp, src = case(tag)
    kw, pkw = config(tag), {}
    if tag == "vr":
        kw.update(track_bodies=vr_track(src), reset_bodies=vr_track(src), full_body_reward=False)
    if tag == "occl":
        pkw = dict(occlusion=src["G_occlusion"].contiguous())
    if tag == "getup":
        pg, cc, ph = getup_inputs(src)
        pkw = dict(point_goal=pg, cycle_counter=cc, cycle_phase=ph)
    plan = make_plan(hp, m, st, smpl_cfg(**kw), **pkw)
    assert plan.obs.shape[1] == exp["obs"].shape[1]
    e.run(plan, variant)
    close(plan.obs, exp["obs"], atol=2e-6, what=f"{tag} obs")
    for k in ("rew", "reward_raw", "reset", "terminate", "amp_obs_buf"):
        close(getattr(plan, k), exp[k], what=f"{tag} {k}")
    if tag == "fut":             # the side buffers keep sample 0 (humanoid_im.py:856-861)
        close(plan.ref_body_pos[0], exp["ref_body_pos"][0], what="fut ref_body_pos env 0")
    else:
        for k in ("ref_body_pos", "ref_body_rot", "ref_body_vel"):
            close(getattr(plan, k), exp[k], what=f"{tag} {k}")
    if tag == "getup":
        k = plan._keep
        for name in ("start_times", "start_offsets", "global_offset"):
            close(k[name], exp[name], what=f"getup {name}")
        close(pkw["point_goal"], exp["point_goal"], what="getup point_goal")
        assert torch.equal(pkw["cycle_counter"].long(), exp["cycle_counter"].long())


# every case through the instantiation phc_env_step launches for it, plus the generic build on the T = 1 cases
@pytest.mark.parametrize("tag,variant", [("A", "smpl"), ("B", "smpl"), ("C", "smpl"), ("occl", "smpl"), ("vr", "smpl"), ("getup", "getup"),
                                         ("fut", "fut"), ("A", "generic"), ("B", "generic"), ("C", "generic"), ("occl", "generic"),
                                         ("vr", "generic")])
def test_kp_kernel_source_vs_reference_golden(emu, tag, variant):
    e, hp = emu
    run_case(e, hp, tag, variant)


def test_kp_chaos_mode_subset():
    """The same emulation with every lane dawdling randomly after each collective (PHC_EMU_CHAOS=1, read when the emulation library
    loads, hence a fresh process), on the cases with the most cross-lane traffic."""
    import subprocess
    if os.environ.get("PHC_EMU_CHAOS") == "1":
        pytest.skip("already inside the chaos run")
    env = dict(os.environ, PHC_EMU_CHAOS="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-p", "no:cacheprovider", "-k",
                        "getup or golden[B-smpl] or golden[vr-generic]"], capture_output=True, text=True, env=env,
                       cwd=os.path.dirname(HERE), timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


def test_kp_task_obs_dim():
    from phc_b200 import build
    build.build()
    lib = _lib.load()
    KP = _lib.PHC_FLAG_TASK_OBS_KP
    assert lib.phc_task_obs_dim_flags(24, 1, KP) == 216
    assert lib.phc_self_obs_dim(24, _lib.PHC_FLAG_ROOT_HEIGHT_OBS) + lib.phc_task_obs_dim_flags(24, 1, KP) == 574
    assert lib.phc_task_obs_dim_flags(3, 3, KP | _lib.PHC_FLAG_UPRIGHT) == 81
    for K, T in ((24, 1), (3, 1), (20, 3), (52, 4)):
        assert lib.phc_task_obs_dim_flags(K, T, 0) == lib.phc_task_obs_dim(K, T)
        assert lib.phc_task_obs_dim_flags(K, T, 0xFFFFFFFF & ~KP) == lib.phc_task_obs_dim(K, T)
    with pytest.raises(NotImplementedError, match="obs_v 5"):
        smpl_cfg(obs_v=5).flags()


@pytest.mark.parametrize("J,getup", [(52, False), (20, True)])
def test_kp_refusals_before_any_launch(J, getup):
    """More than 32 bodies (the strided kernel) and the getup extras on a non-SMPL body count have no keypoint kernel: phc_env_step
    returns PHC_ERR_UNSUPPORTED from its argument checks, which run before anything touches the device (host pointers here)."""
    sys.path.insert(0, os.path.join(HERE, "emu"))
    import host_plan as hp
    from phc_b200 import build
    build.build()
    m = syn.make_motions(4, seed=0, num_bodies=J, min_frames=8, max_frames=12)
    A = 1 + 12 + 9 * (J - 1) + 3
    st = syn.make_env_state(m, 4, seed=0, amp_dim=A, max_progress=4)
    cfg = ops.EnvStepConfig(obs_v=7, key_bodies=[J - 1], reset_bodies=None, dof_subset=None, zero_out_far=getup, cycle_motion=getup)
    extra = dict(point_goal=torch.zeros(4), cycle_counter=torch.zeros(4, dtype=torch.int32), cycle_phase=torch.zeros(4)) if getup else {}
    plan = make_plan(hp, m, st, cfg, **extra)
    assert plan.task_dim == 9 * J
    lib = _lib.load()
    rc = lib.phc_env_step(C.byref(plan.args), None)
    assert rc == -2, rc                                     # PHC_ERR_UNSUPPORTED
    assert b"PHC_FLAG_TASK_OBS_KP" in lib.phc_last_error() or b"keypoint" in lib.phc_last_error()
