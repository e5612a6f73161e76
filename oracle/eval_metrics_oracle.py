"""numpy / fp64 restatement of the imitation evaluation metrics the reference logs at the end of IMAmpAgent's eval sweep: the per-clip
slicing of `_post_step_eval` (phc/learning/im_amp.py:244-363) and smpl_sim's `compute_metrics_lite` with its helpers
`compute_error_vel`, `compute_error_accel` and `p_mpjpe` (VideoPose3D's Procrustes-aligned MPJPE).  smpl_sim is neither in the
reference tree nor installable here, so this is written from the published definitions and pinned by analytic cases and by
scipy's Kabsch solver (tests/test_eval_metrics_cpu.py), not by a reference run.

Conventions of the published code kept here: positions [F, J, 3]; a clip contributes frames [:num_steps - 1]; mpjpe_g / vel / accel on
the global positions, mpjpe_l and mpjpe_pa after subtracting joint 0; every metric is a per-frame mean over the joints, reported in
millimetres; with `concatenate` the per-frame values of all clips are concatenated, so the final `np.mean` weighs clips by frames.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np

METRICS = ("mpjpe_g", "mpjpe_l", "mpjpe_pa", "accel_dist", "vel_dist")


def procrustes(predicted: np.ndarray, target: np.ndarray):
    """Per-frame similarity transform mapping predicted onto target ([F, J, 3] each): rotation R acting on ROW vectors
    (aligned = a * predicted @ R + t), scale a, translation t.  SVD of the normalised cross-covariance with the det(R) = -1 fix."""
    predicted = np.asarray(predicted, dtype=np.float64)
    target = np.asarray(target, dtype=np.float64)
    assert predicted.shape == target.shape and predicted.ndim == 3
    mu_x = target.mean(axis=1, keepdims=True)
    mu_y = predicted.mean(axis=1, keepdims=True)
    x0, y0 = target - mu_x, predicted - mu_y
    norm_x = np.sqrt((x0 ** 2).sum(axis=(1, 2), keepdims=True))
    norm_y = np.sqrt((y0 ** 2).sum(axis=(1, 2), keepdims=True))
    x0, y0 = x0 / norm_x, y0 / norm_y
    h = np.matmul(x0.transpose(0, 2, 1), y0)
    u, s, vt = np.linalg.svd(h)
    v = vt.transpose(0, 2, 1)
    r = np.matmul(v, u.transpose(0, 2, 1))
    sign = np.sign(np.linalg.det(r))                     # a reflection: flip the weakest singular direction
    v[:, :, -1] *= sign[:, None]
    s[:, -1] *= sign
    r = np.matmul(v, u.transpose(0, 2, 1))
    a = s.sum(axis=1)[:, None, None] * norm_x / norm_y
    t = mu_x - a * np.matmul(mu_y, r)
    return r, a, t


def p_mpjpe(predicted: np.ndarray, target: np.ndarray) -> np.ndarray:
    """[F, J, 3] x2 -> [F]: mean over joints of |aligned predicted - target| after the per-frame Procrustes alignment."""
    if predicted.shape[0] == 0:
        return np.zeros(0)
    r, a, t = procrustes(predicted, target)
    aligned = a * np.matmul(np.asarray(predicted, dtype=np.float64), r) + t
    return np.linalg.norm(aligned - target, axis=-1).mean(axis=-1)


def compute_error_vel(joints_gt: np.ndarray, joints_pred: np.ndarray) -> np.ndarray:
    """[F, J, 3] x2 -> [F - 1]: mean over joints of |(p_t - p_{t-1}) - (g_t - g_{t-1})|."""
    vel_gt = joints_gt[1:] - joints_gt[:-1]
    vel_pred = joints_pred[1:] - joints_pred[:-1]
    return np.linalg.norm(vel_pred - vel_gt, axis=2).mean(axis=1) if len(vel_gt) else np.zeros(0)


def compute_error_accel(joints_gt: np.ndarray, joints_pred: np.ndarray) -> np.ndarray:
    """[F, J, 3] x2 -> [F - 2]: mean over joints of the second finite difference of pred minus that of gt."""
    accel_gt = joints_gt[:-2] - 2 * joints_gt[1:-1] + joints_gt[2:]
    accel_pred = joints_pred[:-2] - 2 * joints_pred[1:-1] + joints_pred[2:]
    return np.linalg.norm(accel_pred - accel_gt, axis=2).mean(axis=1) if len(accel_gt) else np.zeros(0)


def compute_metrics_lite(pred_pos_all: Sequence[np.ndarray], gt_pos_all: Sequence[np.ndarray], root_idx: int = 0,
                         concatenate: bool = True) -> Dict[str, np.ndarray]:
    """Per-clip lists of [F_i, J, 3] -> {metric: per-frame values in mm} (concatenated over clips; an empty list gives {})."""
    metrics: Dict[str, List[np.ndarray]] = {}
    for pred, gt in zip(pred_pos_all, gt_pos_all):
        pred = np.asarray(pred, dtype=np.float64)
        gt = np.asarray(gt, dtype=np.float64)
        vals = {"mpjpe_g": np.linalg.norm(gt - pred, axis=2).mean(axis=1) * 1000,
                "vel_dist": compute_error_vel(gt, pred) * 1000,
                "accel_dist": compute_error_accel(gt, pred) * 1000}
        pred_l = pred - pred[:, [root_idx]]
        gt_l = gt - gt[:, [root_idx]]
        vals["mpjpe_pa"] = p_mpjpe(pred_l, gt_l) * 1000
        vals["mpjpe_l"] = np.linalg.norm(pred_l - gt_l, axis=2).mean(axis=1) * 1000
        for k in METRICS:
            metrics.setdefault(k, []).append(vals[k])
    if concatenate:
        return {k: np.concatenate(v) for k, v in metrics.items()}
    return metrics


def slice_batch(pred_steps: np.ndarray, gt_steps: np.ndarray, num_steps: Sequence[int]):
    """One batch of clips as _post_step_eval slices it: stacked steps [S, N, J, 3] -> per-env lists of [:num_steps - 1]."""
    pred = [pred_steps[:(int(i) - 1), e] for e, i in enumerate(num_steps)]
    gt = [gt_steps[:(int(i) - 1), e] for e, i in enumerate(num_steps)]
    return pred, gt


def _mean(v: np.ndarray) -> float:
    return float(v.mean()) if v.size else float("nan")      # numpy's mean of an empty array, without the warning


def eval_info(pred_pos_all: Sequence[np.ndarray], gt_pos_all: Sequence[np.ndarray], terminated: np.ndarray) -> Dict[str, float]:
    """The eight keys _post_step_eval logs for a complete sweep; `terminated` [num_unique] bool, the clip lists already cut to it."""
    terminated = np.asarray(terminated, dtype=bool)
    succ = np.flatnonzero(~terminated).tolist()
    m_all = {k: _mean(v) for k, v in compute_metrics_lite(pred_pos_all, gt_pos_all).items()}
    m_succ = {k: _mean(v) for k, v in compute_metrics_lite([pred_pos_all[i] for i in succ], [gt_pos_all[i] for i in succ]).items()}
    if len(m_succ) == 0:                                      # no clip succeeded
        m_succ = m_all
    return {"eval/success_rate": float(1.0 - terminated.mean()),
            "eval/mpjpe_all": m_all["mpjpe_g"], "eval/mpjpe_succ": m_succ["mpjpe_g"],
            "eval/accel_dist": m_succ["accel_dist"], "eval/vel_dist": m_succ["vel_dist"],
            "eval/mpjpel_all": m_all["mpjpe_l"], "eval/mpjpel_succ": m_succ["mpjpe_l"], "eval/mpjpe_pa": m_succ["mpjpe_pa"]}


def per_env_sums(pred_steps: np.ndarray, gt_steps: np.ndarray, num_steps: Sequence[int]) -> np.ndarray:
    """What the device accumulator row of each env holds after one batch of clips (include/phc_b200.h, phc_eval_metrics_step):
    [N, 8] = sums of the per-frame values of mpjpe_g, mpjpe_l, mpjpe_pa, vel_dist, accel_dist (metres), then the frame counts of
    the first three, of vel_dist and of accel_dist."""
    pred, gt = slice_batch(pred_steps, gt_steps, num_steps)
    rows = []
    for p, g in zip(pred, gt):
        m = compute_metrics_lite([p], [g])
        rows.append([m["mpjpe_g"].sum() / 1000, m["mpjpe_l"].sum() / 1000, m["mpjpe_pa"].sum() / 1000, m["vel_dist"].sum() / 1000,
                     m["accel_dist"].sum() / 1000, len(m["mpjpe_g"]), len(m["vel_dist"]), len(m["accel_dist"])])
    return np.asarray(rows, dtype=np.float64)
