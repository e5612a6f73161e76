"""The imitation evaluation metrics without a GPU: the fp64 oracle (oracle/eval_metrics_oracle.py, compute_metrics_lite and its helpers)
on analytic sequences and against scipy's Kabsch solver, then the kernel source of phc_b200/csrc/eval_metrics.cu through the CPU
emulation of tests/emu against that oracle (J = 20, 24, 52, extend bodies, clip lengths 1-3, a 40-step sequence over two batches of
clips, one subset with every lane dawdling after each collective), and the refusals of the wrapper and of the C ABI."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

from oracle import eval_metrics_oracle as EO                        # noqa: E402
from tests import eval_metrics_cases as EC                          # noqa: E402


def _seq(seed, F=6, J=24):
    rng = np.random.default_rng(seed)
    return rng, rng.standard_normal((F, J, 3)) * 0.3 + np.array([0.0, 0.0, 0.9])


# ---- the oracle on analytic sequences -----------------------------------------------------------------------------------
def test_similarity_transform_has_zero_pa_error():
    rng, gt = _seq(0)
    R = EC.rotations(rng, gt.shape[0])
    s = rng.uniform(0.5, 2.0, (gt.shape[0], 1, 1))
    pred = s * np.einsum("fab,fjb->fja", R, gt) + rng.standard_normal((gt.shape[0], 1, 3))
    m = EO.compute_metrics_lite([pred], [gt])
    assert np.all(m["mpjpe_pa"] < 1e-9) and np.all(m["mpjpe_g"] > 1.0)
    # the recovered transform is the inverse one: row-vector R_o = R (column form R^T maps pred back onto gt)
    r, a, _ = EO.procrustes(pred, gt)
    np.testing.assert_allclose(r, R, atol=1e-9)
    np.testing.assert_allclose(a[:, 0, 0], 1.0 / s[:, 0, 0], rtol=1e-9)


def test_mirrored_pred_has_the_sign_fixed_error():
    """A reflection cannot be undone by a proper rotation: the PA error is positive and equals that of the best proper rotation
    (scipy's Kabsch) with the optimal scale -- the det(R) = -1 fix of p_mpjpe."""
    from scipy.spatial.transform import Rotation
    _, gt = _seq(1)
    pred = gt * np.array([-1.0, 1.0, 1.0])
    got = EO.p_mpjpe(pred, gt)
    for f in range(gt.shape[0]):
        x0, y0 = gt[f] - gt[f].mean(0), pred[f] - pred[f].mean(0)
        rot, _ = Rotation.align_vectors(x0, y0)
        ry = rot.apply(y0)
        a = (x0 * ry).sum() / (y0 ** 2).sum()
        exp = np.linalg.norm(a * ry - x0, axis=1).mean()
        assert exp > 1e-2
        assert abs(got[f] - exp) < 1e-9 * max(1.0, exp)
    # without the fix (an improper "rotation" allowed) the error would be zero
    u, s, vt = np.linalg.svd(np.matmul((gt - gt.mean(1, keepdims=True)).transpose(0, 2, 1), pred - pred.mean(1, keepdims=True)))
    assert np.all(np.linalg.det(np.matmul(vt.transpose(0, 2, 1), u.transpose(0, 2, 1))) < 0)


def test_constant_offset_has_no_velocity_or_acceleration_error():
    rng, gt = _seq(2)
    c = rng.standard_normal(3) * 0.1
    m = EO.compute_metrics_lite([gt + c], [gt])
    assert np.all(m["vel_dist"] < 1e-9) and np.all(m["accel_dist"] < 1e-9) and np.all(m["mpjpe_l"] < 1e-9)
    np.testing.assert_allclose(m["mpjpe_g"], np.linalg.norm(c) * 1000, rtol=1e-12)
    cj = rng.standard_normal((gt.shape[1], 3)) * 0.1               # per-joint offsets: still no velocity error, but a local one
    m = EO.compute_metrics_lite([gt + cj], [gt])
    assert np.all(m["vel_dist"] < 1e-9) and np.all(m["accel_dist"] < 1e-9) and np.all(m["mpjpe_l"] > 1.0)
    assert m["vel_dist"].shape == (gt.shape[0] - 1,) and m["accel_dist"].shape == (gt.shape[0] - 2,)


def test_constant_velocity_drift():
    rng, gt = _seq(3)
    v = rng.standard_normal(3) * 0.05
    pred = gt + v * np.arange(gt.shape[0])[:, None, None]
    m = EO.compute_metrics_lite([pred], [gt])
    assert np.all(m["accel_dist"] < 1e-9)
    np.testing.assert_allclose(m["vel_dist"], np.linalg.norm(v) * 1000, rtol=1e-12)


def test_oracle_rotation_matches_scipy_kabsch():
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(4)
    gt = rng.standard_normal((20, 24, 3))
    pred = gt + 0.3 * rng.standard_normal(gt.shape)
    r, _, _ = EO.procrustes(pred, gt)
    for f in range(gt.shape[0]):
        rot, _ = Rotation.align_vectors(gt[f] - gt[f].mean(0), pred[f] - pred[f].mean(0))
        np.testing.assert_allclose(r[f], rot.as_matrix().T, atol=1e-9)          # row-vector convention: pred @ R
        assert abs(np.linalg.det(r[f]) - 1.0) < 1e-9


def test_eval_info_frame_weighting_and_fallback():
    """Frames are weighted, not clips; "succ" falls back to "all" without a successful clip; a metric without frames is NaN."""
    rng = np.random.default_rng(5)
    clips_g = [rng.standard_normal((F, 24, 3)) for F in (2, 10)]
    clips_p = [g + 0.1 for g in clips_g]
    clips_p[0] = clips_g[0] + 0.5
    info = EO.eval_info(clips_p, clips_g, np.array([False, False]))
    exp = (2 * np.linalg.norm([0.5] * 3) + 10 * np.linalg.norm([0.1] * 3)) / 12 * 1000
    assert abs(info["eval/mpjpe_all"] - exp) < 1e-9 and info["eval/success_rate"] == 1.0
    info = EO.eval_info(clips_p, clips_g, np.array([True, True]))
    assert info["eval/mpjpe_succ"] == info["eval/mpjpe_all"] and info["eval/success_rate"] == 0.0
    info = EO.eval_info(clips_p, clips_g, np.array([True, False]))
    assert abs(info["eval/mpjpe_succ"] - np.linalg.norm([0.1] * 3) * 1000) < 1e-9
    info = EO.eval_info([clips_p[0]], [clips_g[0]], np.array([False]))                       # 2 frames: no acceleration
    assert np.isnan(info["eval/accel_dist"]) and not np.isnan(info["eval/vel_dist"])


# ---- the kernel source under the CPU emulation ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    import shutil
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    import eval_metrics_emu
    return eval_metrics_emu.EmuEvalMetrics(eval_metrics_emu.build(str(tmp_path_factory.mktemp("emu_eval_metrics"))))


@pytest.mark.parametrize("case", EC.CASES, ids=[c[0] for c in EC.CASES])
def test_emulated_kernel_matches_the_oracle(emu, case):
    _, n, J, B, S = case
    state, gt, ns = EC.make_case(n, J, B, S, seed=J + B)
    acc, _ = EC.run(emu.step, state, gt, ns, J)
    exp = EC.expected(state, gt, ns, J)
    assert exp[:3, 5].tolist() == [0, 1, 2] and exp[2, 6] == 1 and exp[2, 7] == 0          # clip lengths 1, 2, 3
    EC.compare(acc, exp)


@pytest.mark.parametrize("J", [20, 52])
def test_emulated_kernel_undoes_a_known_similarity(emu, J):
    """pred = s R gt + t per frame: the aligned error vanishes (a transposed rotation would not)."""
    state, gt, ns = EC.make_case(5, J, J, 5, seed=J, num_steps=[9] * 5, kind="similar")
    acc, _ = EC.run(emu.step, state, gt, ns, J)
    got = acc.numpy()
    assert np.all(got[:, 5] == 5) and np.all(got[:, 2] / got[:, 5] < 2e-6) and np.all(got[:, 0] / got[:, 5] > 1e-2)
    EC.compare(acc, EC.expected(state, gt, ns, J))


def test_emulated_kernel_40_steps_two_batches(emu):
    """40 steps as two batches of clips (25 + 15 steps, t restarting at 0, the ring kept as it is): per-env sums and counts of
    each batch against the oracle's slices."""
    n, J = 6, 24
    state, gt, ns = EC.make_case(n, J, J, 40, seed=40, num_steps=[1, 2, 3, 20, 26, 40])
    acc, ring = EC.run(emu.step, state[:25], gt[:25], ns, J)
    EC.compare(acc, EC.expected(state[:25], gt[:25], ns, J))
    acc2, _ = EC.run(emu.step, state[25:], gt[25:], ns, J, ring=ring)
    EC.compare(acc2, EC.expected(state[25:], gt[25:], ns, J))
    assert acc[5, 5] == 25 and acc[5, 7] == 23 and acc2[5, 5] == 15 and acc2[0, 5] == 0


def test_eval_metrics_chaos_mode_subset():
    """The same emulation with every lane dawdling randomly after each collective (PHC_EMU_CHAOS=1, read when the emulation library
    loads, hence a fresh process)."""
    import subprocess
    if os.environ.get("PHC_EMU_CHAOS") == "1":
        pytest.skip("already inside the chaos run")
    env = dict(os.environ, PHC_EMU_CHAOS="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-p", "no:cacheprovider", "-k",
                        "emulated_kernel_matches and smpl_ext or known_similarity and 20"], capture_output=True, text=True, env=env,
                       cwd=os.path.dirname(HERE), timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


# ---- refusals -----------------------------------------------------------------------------------------------------------
def test_wrapper_refuses_cpu_tensors_and_too_many_bodies():
    from phc_b200 import ops
    n, J = 4, 24
    args = lambda J: (torch.zeros(n, J, 3), torch.zeros(n, J, 3), torch.ones(n, dtype=torch.int32), 0, torch.zeros(2, n, J, 3),
                      torch.zeros(n, 8, dtype=torch.float64))
    with pytest.raises(ops.PhcError):
        ops.eval_metrics_step(*args(J))
    with pytest.raises(ValueError, match="1..64"):
        ops.eval_metrics_step(*args(65))


def test_c_abi_refuses_bad_input():
    """phc_eval_metrics_step validates before it launches: J > 64, x / y / z not contiguous, n <= 0, short strides."""
    from phc_b200 import _lib
    lib = _lib.load()
    p = 256                                              # never dereferenced: every call below is refused first
    ok = dict(env_stride=24 * 13, body_stride=13, coord_stride=1, t=0, n=4, J=24)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.phc_eval_metrics_step(p, a["env_stride"], a["body_stride"], a["coord_stride"], p, p, a["t"], a["n"], a["J"], p, p, None)
    for bad in (dict(J=65, env_stride=65 * 13), dict(J=0), dict(coord_stride=2), dict(n=0), dict(n=-3), dict(body_stride=2),
                dict(env_stride=23 * 13), dict(t=-1)):
        assert call(**bad) == -1, bad
        assert lib.phc_last_error().decode().startswith("phc_eval_metrics_step")
