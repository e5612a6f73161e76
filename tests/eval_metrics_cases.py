"""Shared cases of the evaluation-metrics tests (tests/test_eval_metrics_cpu.py through the CPU emulation, tests/test_gpu_eval_metrics.py
through the C ABI): seeded eval-step sequences of simulated and reference body positions, a driver that feeds them step by step to a
phc_eval_metrics_step implementation, and the oracle's per-env sums for the same frames."""
import numpy as np
import torch

from oracle import eval_metrics_oracle as EO

EO_FIELDS = 8                                      # PHC_EVAL_ACC_FIELDS

# (name, n envs, J, bodies per env, steps): J = 20 (H1), 24 (SMPL), 52 (SMPL-X); n not a multiple of the 4 envs per CTA; bodies > J
# (extend bodies after the J simulated ones)
CASES = [("h1", 7, 20, 23, 12), ("smpl", 10, 24, 24, 12), ("smplx", 5, 52, 52, 9), ("smpl_ext", 6, 24, 27, 10)]


def rotations(rng, n):
    """n random proper rotation matrices (QR of Gaussian matrices, det fixed to +1)."""
    q, r = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    q = q * np.sign(np.diagonal(r, axis1=1, axis2=2))[:, None, :]
    q[np.linalg.det(q) < 0, :, 0] *= -1
    return q


def make_case(n, J, bodies, steps, seed, num_steps=None, kind="noisy"):
    """-> state [steps, n, bodies, 13] fp32 (positions in columns 0:3 of the first J records, the rest filler), gt [steps, n, J, 3] fp32,
    num_steps [n] int32.  kind "noisy": pred = gt + a smooth per-joint drift + cm noise; "similar": pred = s R gt + t per frame."""
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((n, J, 3)) * 0.3 + np.array([0.0, 0.0, 0.9])
    vel = rng.standard_normal((n, J, 3)) * 0.02
    tt = np.arange(steps, dtype=np.float64)[:, None, None, None]
    gt = base[None] + vel[None] * tt + 0.01 * np.sin(0.3 * tt + rng.standard_normal((1, n, J, 3)))
    if kind == "similar":
        R = rotations(rng, steps * n).reshape(steps, n, 3, 3)
        s = rng.uniform(0.5, 2.0, (steps, n, 1, 1))
        tr = rng.standard_normal((steps, n, 1, 3))
        pred = s * np.einsum("tnab,tnjb->tnja", R, gt) + tr
    else:
        drift = rng.standard_normal((n, J, 3)) * 0.01
        pred = gt + drift[None] * np.sqrt(tt + 1.0) + rng.standard_normal((steps, n, J, 3)) * 0.02
    state = rng.standard_normal((steps, n, bodies, 13)).astype(np.float32)
    state[:, :, :J, 0:3] = pred
    if num_steps is None:                          # lengths 1, 2 and 3 (0, 1 and 2 counted frames) and longer ones, some past `steps`
        num_steps = np.concatenate([[1, 2, 3], rng.integers(4, steps + 4, max(0, n - 3))])[:n]
    return torch.from_numpy(state), torch.from_numpy(gt.astype(np.float32)), torch.as_tensor(np.asarray(num_steps), dtype=torch.int32)


def run(step_fn, state, gt, num_steps, J, ring=None, acc=None, t0=0):
    """Feed steps t0, t0 + 1, ... to step_fn(body_pos_view, gt, num_steps, t, ring, acc); returns (acc, ring)."""
    S, n = gt.shape[0], gt.shape[1]
    dev = state.device
    ring = torch.full((2, n, J, 3), float("nan"), device=dev) if ring is None else ring      # the kernel must not read unwritten slots
    acc = torch.zeros(n, EO_FIELDS, dtype=torch.float64, device=dev) if acc is None else acc
    for t in range(S):
        step_fn(state[t][:, :J, 0:3], gt[t].contiguous(), num_steps, t0 + t, ring, acc)
    return acc, ring



def expected(state, gt, num_steps, J):
    pred = state[..., :J, 0:3].double().cpu().numpy()
    return EO.per_env_sums(pred, gt.double().cpu().numpy(), num_steps.cpu().numpy())


def compare(acc, exp, rtol=1e-4, atol_mm=1e-3):
    """Counts exactly; per-env means of every metric in mm within rtol / atol; an env without counted frames has zero sums."""
    got = acc.cpu().numpy()
    assert np.array_equal(got[:, 5:], exp[:, 5:]), (got[:, 5:], exp[:, 5:])
    cnt = exp[:, [5, 5, 5, 6, 7]]
    zero = cnt == 0
    assert np.all(got[:, :5][zero] == 0)
    g = got[:, :5][~zero] / cnt[~zero] * 1000
    e = exp[:, :5][~zero] / cnt[~zero] * 1000
    np.testing.assert_allclose(g, e, rtol=rtol, atol=atol_mm)
