"""Torch-facing wrappers over the C ABI (include/phc_b200.h).  PyTorch only provides device memory and streams:
every function here validates its tensors, hands `data_ptr()`s plus the current CUDA stream to libphc_b200.so and
returns torch tensors that the caller (or this module) allocated.  There is no non-CUDA path.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from ._lib import (PHC_FLAG_EARLY_TERM, PHC_FLAG_LOCAL_ROOT_OBS, PHC_FLAG_NO_COLLISION, PHC_FLAG_POWER_REWARD,
                   PHC_FLAG_ROOT_HEIGHT_OBS, PHC_FLAG_TERM_USE_MEAN, PHC_FLAG_UPRIGHT, PhcError)

__all__ = ["PackedMotionLib", "pack_motion_lib", "load_motion_tables", "motion_state", "EnvStepConfig", "EnvStepPlan", "amp_obs_demo",
           "gae", "adv_norm", "PhcError"]


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _req(t: torch.Tensor, dtype, name: str, device=None) -> torch.Tensor:
    if not torch.is_tensor(t):
        raise TypeError(f"{name}: expected a torch tensor")
    if not t.is_cuda:
        raise PhcError(f"{name}: phc_b200 runs on CUDA tensors only (got {t.device}); there is no CPU fallback")
    if t.dtype != dtype:
        raise TypeError(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name}: must be contiguous")
    if device is not None and t.device != device:
        raise ValueError(f"{name}: on {t.device}, expected {device}")
    return t


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


# ------------------------------------------------------------------------------------------------------------
# motion library
# ------------------------------------------------------------------------------------------------------------
@dataclass
class PackedMotionLib:
    """Packed device copy of the MotionLib frame tables (PhcMotionLib in the header).  Keeps the tensors alive."""
    frames_body: torch.Tensor
    frames_joint: Optional[torch.Tensor]
    lengths: torch.Tensor
    dts: torch.Tensor
    num_frames: torch.Tensor
    length_starts: torch.Tensor
    num_bodies: int
    c: _lib.PhcMotionLib = field(default=None, repr=False)
    num_ext_bodies: int = 0          # robots: "extend" bodies stored as records J..J+E-1
    num_dofs: int = 0                # robots: hinge dofs (0 = SMPL spherical joints, D = 3(J-1))

    @property
    def dofs(self) -> int:
        return self.num_dofs if self.num_dofs > 0 else 3 * (self.num_bodies - 1)

    @property
    def device(self):
        return self.frames_body.device

    @property
    def num_motions(self) -> int:
        return int(self.lengths.shape[0])


def pack_motion_lib(gts, grs, gvs, gavs, lrs, dvs, lengths, num_frames, dts, length_starts) -> PackedMotionLib:
    """phc_motion_pack: the reference's separate [F,J,*] tables -> 16-byte aligned per-frame records."""
    lib = _lib.load()
    dev = gts.device
    f32, i64 = torch.float32, torch.int64
    gts, grs = _req(gts, f32, "gts"), _req(grs, f32, "grs", dev)
    gvs, gavs = _req(gvs, f32, "gvs", dev), _req(gavs, f32, "gavs", dev)
    F, J = int(gts.shape[0]), int(gts.shape[1])
    assert grs.shape == (F, J, 4) and gvs.shape == (F, J, 3) and gavs.shape == (F, J, 3)
    joint = lrs is not None and dvs is not None
    if joint:
        lrs, dvs = _req(lrs, f32, "lrs", dev), _req(dvs, f32, "dvs", dev)
        assert lrs.shape == (F, J, 4) and dvs.shape == (F, J - 1, 3)
    bs, js = lib.phc_motion_body_stride(J), lib.phc_motion_joint_stride(J)
    fb = torch.empty(F, bs, dtype=f32, device=dev)
    fj = torch.empty(F, js, dtype=f32, device=dev) if joint else None
    with torch.cuda.device(dev):
        _lib.check(lib.phc_motion_pack(gts.data_ptr(), grs.data_ptr(), gvs.data_ptr(), gavs.data_ptr(),
                                       _ptr(lrs) if joint else None, _ptr(dvs) if joint else None, F, J,
                                       fb.data_ptr(), _ptr(fj), _stream()), "phc_motion_pack")
    lengths = _req(lengths.contiguous(), f32, "lengths", dev)
    dts = _req(dts.contiguous(), f32, "dts", dev)
    num_frames = _req(num_frames.contiguous(), i64, "num_frames", dev)
    length_starts = _req(length_starts.contiguous(), i64, "length_starts", dev)
    c = _lib.PhcMotionLib(fb.data_ptr(), _ptr(fj), lengths.data_ptr(), dts.data_ptr(), num_frames.data_ptr(),
                          length_starts.data_ptr(), F, int(lengths.shape[0]), J, bs, js)
    return PackedMotionLib(fb, fj, lengths, dts, num_frames, length_starts, J, c)


def pack_robot_motion_lib(gts_t, grs_t, gvs_t, gavs_t, dof_pos, dof_vel, num_bodies: int, lengths, num_frames, dts,
                          length_starts) -> PackedMotionLib:
    """Hinge-joint robots (H1 / G1, phc/utils/motion_lib_real.py): the *_t tables hold all J + E bodies (J simulated ones
    first, then the "extend" bodies), dof_pos / dof_vel are [F, D].  Body records via phc_motion_pack(J + E), joint records via
    phc_motion_pack_dofs."""
    lib = _lib.load()
    dev = gts_t.device
    f32, i64 = torch.float32, torch.int64
    gts_t, grs_t = _req(gts_t, f32, "gts_t"), _req(grs_t, f32, "grs_t", dev)
    gvs_t, gavs_t = _req(gvs_t, f32, "gvs_t", dev), _req(gavs_t, f32, "gavs_t", dev)
    dof_pos, dof_vel = _req(dof_pos, f32, "dof_pos", dev), _req(dof_vel, f32, "dof_vel", dev)
    F, JE = int(gts_t.shape[0]), int(gts_t.shape[1])
    J, E, D = int(num_bodies), JE - int(num_bodies), int(dof_pos.shape[1])
    assert 0 <= E <= _lib.PHC_MAX_EXT_BODIES and grs_t.shape == (F, JE, 4) and gvs_t.shape == (F, JE, 3) and gavs_t.shape == (F, JE, 3)
    assert dof_pos.shape == (F, D) and dof_vel.shape == (F, D)
    bs, js = lib.phc_motion_body_stride(JE), lib.phc_motion_dof_stride(D)
    fb = torch.empty(F, bs, dtype=f32, device=dev)
    fj = torch.empty(F, js, dtype=f32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.phc_motion_pack(gts_t.data_ptr(), grs_t.data_ptr(), gvs_t.data_ptr(), gavs_t.data_ptr(), None, None, F, JE,
                                       fb.data_ptr(), None, _stream()), "phc_motion_pack")
        _lib.check(lib.phc_motion_pack_dofs(dof_pos.data_ptr(), dof_vel.data_ptr(), F, D, fj.data_ptr(), _stream()), "phc_motion_pack_dofs")
    lengths = _req(lengths.contiguous(), f32, "lengths", dev)
    dts = _req(dts.contiguous(), f32, "dts", dev)
    num_frames = _req(num_frames.contiguous(), i64, "num_frames", dev)
    length_starts = _req(length_starts.contiguous(), i64, "length_starts", dev)
    c = _lib.PhcMotionLib(fb.data_ptr(), fj.data_ptr(), lengths.data_ptr(), dts.data_ptr(), num_frames.data_ptr(),
                          length_starts.data_ptr(), F, int(lengths.shape[0]), J, bs, js, E, D)
    return PackedMotionLib(fb, fj, lengths, dts, num_frames, length_starts, J, c, E, D)


def load_motion_tables(pose_quat_global: torch.Tensor, root_trans: torch.Tensor, offsets: torch.Tensor, parents: torch.Tensor,
                       num_frames: torch.Tensor, fps: torch.Tensor, heading: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """phc_motion_load: concatenated on-disk clip arrays (float64, on the device) -> the reference's float32 tables
    gts / grs / lrs / gvs / gavs / dvs plus lengths / dts / length_starts (motion_lib_base.py:262-313)."""
    lib = _lib.load()
    f64, i64 = torch.float64, torch.int64
    q = _req(pose_quat_global, f64, "pose_quat_global")
    dev = q.device
    F, J = int(q.shape[0]), int(q.shape[1])
    t = _req(root_trans, f64, "root_trans", dev)
    off = _req(offsets, f64, "offsets", dev)
    par = _req(parents, torch.int32, "parents", dev)
    nf = _req(num_frames, i64, "num_frames", dev)
    fps = _req(fps, f64, "fps", dev)
    M = int(nf.shape[0])
    assert q.shape == (F, J, 4) and t.shape == (F, 3) and off.shape == (M, J, 3) and par.shape == (J,) and fps.shape == (M,)
    if heading is not None:
        heading = _req(heading, f64, "heading", dev)
        assert heading.shape == (M,)
    starts = (torch.cumsum(nf, 0) - nf).contiguous()
    f32 = torch.float32
    out = dict(gts=torch.empty(F, J, 3, dtype=f32, device=dev), grs=torch.empty(F, J, 4, dtype=f32, device=dev),
               lrs=torch.empty(F, J, 4, dtype=f32, device=dev), gvs=torch.empty(F, J, 3, dtype=f32, device=dev),
               gavs=torch.empty(F, J, 3, dtype=f32, device=dev), dvs=torch.empty(F, J - 1, 3, dtype=f32, device=dev))
    ws = torch.empty(max(16, int(lib.phc_motion_load_workspace_bytes(F, J))), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.phc_motion_load(q.data_ptr(), t.data_ptr(), off.data_ptr(), par.data_ptr(), _ptr(heading),
                                       starts.data_ptr(), nf.data_ptr(), fps.data_ptr(), F, M, J, out["gts"].data_ptr(),
                                       out["grs"].data_ptr(), out["lrs"].data_ptr(), out["gvs"].data_ptr(),
                                       out["gavs"].data_ptr(), out["dvs"].data_ptr(), ws.data_ptr(), _stream()),
                   "phc_motion_load")
    ws.record_stream(torch.cuda.current_stream(dev))
    out["num_frames"] = nf
    out["length_starts"] = starts
    out["dts"] = (1.0 / fps).to(f32)                                      # curr_dt = 1.0 / motion_fps
    out["lengths"] = ((1.0 / fps) * (nf - 1).to(f64)).to(f32)            # curr_len = 1.0 / motion_fps * (num_frames - 1)
    return out


_MS_KEYS = {"rg_pos": 3, "rb_rot": 4, "body_vel": 3, "body_ang_vel": 3}


def motion_state(mlib: PackedMotionLib, motion_ids: torch.Tensor, motion_times: torch.Tensor,
                 offset: Optional[torch.Tensor] = None, want_dof: bool = True) -> Dict[str, torch.Tensor]:
    """MotionLibBase.get_motion_state (motion_lib_base.py:437-520) on the packed tables."""
    lib = _lib.load()
    dev = mlib.device
    ids = _req(motion_ids, torch.int64, "motion_ids", dev)
    times = _req(motion_times, torch.float32, "motion_times", dev)
    n, J = int(ids.shape[0]), mlib.num_bodies
    if offset is not None:
        offset = _req(offset, torch.float32, "offset", dev)
        assert offset.shape == (n, 3)
    out = {k: torch.empty(n, J, w, dtype=torch.float32, device=dev) for k, w in _MS_KEYS.items()}
    for k, w in (("root_pos", 3), ("root_rot", 4), ("root_vel", 3), ("root_ang_vel", 3)):
        out[k] = torch.empty(n, w, dtype=torch.float32, device=dev)
    if want_dof:
        if mlib.frames_joint is None:
            raise PhcError("motion_state: dof_pos/dof_vel need the joint table (lrs/dvs) in the packed library")
        out["dof_pos"] = torch.empty(n, mlib.dofs, dtype=torch.float32, device=dev)
        out["dof_vel"] = torch.empty(n, mlib.dofs, dtype=torch.float32, device=dev)
    if mlib.num_ext_bodies > 0:          # robots: rg_pos_t / rg_rot_t / body_vel_t / body_ang_vel_t over all J + E bodies
        JE = J + mlib.num_ext_bodies
        for k, w in (("rg_pos_t", 3), ("rg_rot_t", 4), ("body_vel_t", 3), ("body_ang_vel_t", 3)):
            out[k] = torch.empty(n, JE, w, dtype=torch.float32, device=dev)
    co = _lib.PhcMotionStateOut(**{k: _ptr(out.get(k)) for k, _ in _lib.PhcMotionStateOut._fields_})
    with torch.cuda.device(dev):
        _lib.check(lib.phc_motion_state(C.byref(mlib.c), ids.data_ptr(), times.data_ptr(), _ptr(offset), n,
                                        C.byref(co), _stream()), "phc_motion_state")
    return out


# ------------------------------------------------------------------------------------------------------------
# fused env step
# ------------------------------------------------------------------------------------------------------------
@dataclass
class EnvStepConfig:
    """Static configuration of the fused step (what HumanoidIm reads from cfg at construction time)."""
    dt: float = 1.0 / 30.0
    time_steps: int = 1
    traj_dt: float = 0.0
    upright: bool = True
    local_root_obs: bool = True
    root_height_obs: bool = True
    power_reward: bool = True
    power_coef: float = 0.0005
    early_term: bool = True
    no_collision: bool = False
    term_use_mean: bool = False
    k_pos: float = 100.0
    k_rot: float = 10.0
    k_vel: float = 0.1
    k_ang_vel: float = 0.1
    w_pos: float = 0.5
    w_rot: float = 0.3
    w_vel: float = 0.1
    w_ang_vel: float = 0.1
    key_bodies: Sequence[int] = (7, 3, 22, 17)
    reset_bodies: Optional[Sequence[int]] = None         # None = all bodies
    term_dist: float = 0.25                              # or a per-body sequence of length J
    dof_subset: Optional[Sequence[int]] = None           # dof indices kept in the AMP obs (whole joints); None = all
    amp_steps: int = 10
    # robots (cfg.robot.extend_config, humanoid_im.py:74-82): parent body index and position in the parent frame of every
    # "extend" body; must match the E extra records of the packed motion library
    ext_parents: Sequence[int] = ()
    ext_pos: Sequence[Sequence[float]] = ()
    # env_im_getup_mcp.yaml (the configuration HumanoidImMCP trains in)
    zero_out_far: bool = False         # env.zero_out_far (with zero_out_far_train False)
    close_distance: float = 0.25       # env.close_distance
    far_distance: float = 3.0          # env.far_distance
    cycle_motion: bool = False         # env.cycle_motion
    max_episode_length: int = 300      # env.episode_length
    specialise: bool = True            # False: PHC_FLAG_NO_SPECIALISE (always the generic kernel instantiation)
    # env.trackBodies / env.full_body_reward (humanoid_im.py:64-66, :926-935; env_vr.yaml): body ids whose reference enters the task
    # observation (None = all) and whether the tracking reward still averages over every body
    track_bodies: Optional[Sequence[int]] = None
    full_body_reward: bool = True
    # env.obs_v: 6 = compute_imitation_observations_v6 (24 columns per tracked body and sample), 7 = the keypoint-only v7 of the
    # keypoint models (9 columns: position / velocity differences and reference positions, humanoid_im.py:1362-1393)
    obs_v: int = 6

    def flags(self) -> int:
        if self.obs_v not in (6, 7):
            raise NotImplementedError(f"obs_v {self.obs_v}: only the task observations v6 and v7 (keypoints) are built")
        f = 0
        for on, bit in ((self.upright, PHC_FLAG_UPRIGHT), (self.local_root_obs, PHC_FLAG_LOCAL_ROOT_OBS),
                        (self.root_height_obs, PHC_FLAG_ROOT_HEIGHT_OBS), (self.power_reward, PHC_FLAG_POWER_REWARD),
                        (self.early_term, PHC_FLAG_EARLY_TERM), (self.no_collision, PHC_FLAG_NO_COLLISION),
                        (self.term_use_mean, PHC_FLAG_TERM_USE_MEAN), (self.zero_out_far, _lib.PHC_FLAG_ZERO_OUT_FAR),
                        (self.cycle_motion, _lib.PHC_FLAG_CYCLE_MOTION), (not self.specialise, _lib.PHC_FLAG_NO_SPECIALISE),
                        (not self.full_body_reward, _lib.PHC_FLAG_SUBSET_REWARD), (self.obs_v == 7, _lib.PHC_FLAG_TASK_OBS_KP)):
            if on:
                f |= bit
        return f

    def amp_joint_list(self, num_bodies: int):
        if self.dof_subset is None:
            return list(range(num_bodies - 1))
        ds = [int(x) for x in self.dof_subset]
        if len(ds) % 3 or any(ds[i] % 3 or ds[i + 1] != ds[i] + 1 or ds[i + 2] != ds[i] + 2 for i in range(0, len(ds), 3)):
            raise ValueError("dof_subset must be made of whole joints (consecutive dof triples), as humanoid.py:409-413 builds it")
        return [d // 3 for d in ds[::3]]


class EnvStepPlan:
    """A bound launch of phc_env_step: all pointers are captured once (the simulator tensors and the task buffers are
    persistent, exactly as in the reference), `run()` only launches.  Output buffers not supplied are allocated."""

    def __init__(self, cfg: EnvStepConfig, mlib: PackedMotionLib, body_state: torch.Tensor, dof_state: torch.Tensor,
                 dof_force: Optional[torch.Tensor], progress: torch.Tensor, motion_ids: torch.Tensor,
                 start_times: torch.Tensor, start_offsets: torch.Tensor, global_offset: torch.Tensor,
                 cycle_counter: Optional[torch.Tensor] = None, obs: Optional[torch.Tensor] = None,
                 rew: Optional[torch.Tensor] = None, reward_raw: Optional[torch.Tensor] = None,
                 reset: Optional[torch.Tensor] = None, terminate: Optional[torch.Tensor] = None,
                 amp_obs_buf: Optional[torch.Tensor] = None, amp_hist_in: Optional[torch.Tensor] = None,
                 amp_shift: bool = True, with_amp: bool = True, with_ref_buffers: bool = False,
                 only_where: Optional[torch.Tensor] = None, obs_only: bool = False, amp_ring: bool = False,
                 ref_cache: Optional[torch.Tensor] = None, reward_from_cache: bool = False,
                 point_goal: Optional[torch.Tensor] = None, cycle_phase: Optional[torch.Tensor] = None,
                 with_eval_extras: bool = False, ring_head_dev: Optional[torch.Tensor] = None, occlusion: Optional[torch.Tensor] = None,
                 shape_params: Optional[torch.Tensor] = None, limb_weights: Optional[torch.Tensor] = None, amp_current: bool = False):
        """ref_cache: [N, body_stride] pose cache (PhcStepArgs.ref_cache): every run() stores the reference pose interpolated
        for the first observation sample; reward_from_cache=True makes run() take the reward-time reference pose from it
        (valid for HumanoidIm's step / reset sequence, see include/phc_b200.h).
        amp_ring=True: `amp_obs_buf` is a ring -- each run() writes only the newest vector into slot `ring_head`
        (advance with advance_ring() before the step); otherwise the reference's window shift is done in the kernel.
        amp_current=True (with obs_only): the launch also writes the AMP vector of the current simulator state into the newest slot
        (PHC_FLAG_AMP_CURRENT, the get-up reset path); the window is not shifted.
        ring_head_dev: int32 [1] device tensor holding the ring head (PhcStepArgs.ring_head): the slot is then read on the device and
        advance_ring() is a one-thread kernel, so consecutive steps differ in nothing the host passes (CUDA-graph capturable)."""
        lib = _lib.load()
        self._lib = lib
        self.cfg, self.mlib = cfg, mlib
        dev = mlib.device
        self.device = dev
        f32, i64 = torch.float32, torch.int64
        J = mlib.num_bodies
        D = mlib.dofs
        body_state = _req(body_state, f32, "body_state", dev)
        N, bpe = int(body_state.shape[0]), int(body_state.shape[1])
        assert body_state.shape[2] == 13 and bpe >= J
        dof_state = _req(dof_state, f32, "dof_state", dev)
        assert dof_state.shape == (N, D, 2)
        if cfg.power_reward:
            dof_force = _req(dof_force, f32, "dof_force", dev)
            assert dof_force.shape == (N, D)
        self.N, self.J = N, J
        flags = cfg.flags() | (_lib.PHC_FLAG_OBS_ONLY if obs_only else 0)
        if amp_current:
            assert obs_only and with_amp, "amp_current is an option of the observation-only launch with an AMP buffer"
            flags |= _lib.PHC_FLAG_AMP_CURRENT
            amp_shift = False
        if reward_from_cache:
            assert ref_cache is not None and not obs_only
            flags |= _lib.PHC_FLAG_REWARD_FROM_CACHE
        # occlusion [N, K] uint8 / bool (random_occlu_idx), shape_params [N, ns] / limb_weights [N, nl]: the has_shape_obs /
        # has_limb_weight_obs tails of the self observation (humanoid.py:2043-2047)
        K = J if cfg.track_bodies is None else len(cfg.track_bodies)
        ns = 0 if shape_params is None else int(shape_params.shape[1])
        nl = 0 if limb_weights is None else int(limb_weights.shape[1])
        self.self_dim = lib.phc_self_obs_dim(J, flags) + ns + nl
        self.task_dim = lib.phc_task_obs_dim_flags(K, cfg.time_steps, flags)
        self.obs_dim = self.self_dim + self.task_dim
        robot = mlib.num_dofs > 0
        joints = [] if robot else cfg.amp_joint_list(J)
        self.amp_dim = (lib.phc_amp_obs_dim_robot(D, len(cfg.key_bodies), flags) if robot
                        else lib.phc_amp_obs_dim(len(joints), len(cfg.key_bodies), flags))
        E = mlib.num_ext_bodies
        if len(cfg.ext_parents) != E or len(cfg.ext_pos) != E:
            raise PhcError(f"EnvStepConfig.ext_parents / ext_pos must list the {E} extend bodies of the motion library")
        rw = 5 if cfg.power_reward else 4

        def out(t, shape, dtype, name):
            if t is None:
                return torch.zeros(shape, dtype=dtype, device=dev)
            t = _req(t, dtype, name, dev)
            assert tuple(t.shape) == tuple(shape), f"{name}: shape {tuple(t.shape)} != {tuple(shape)}"
            return t

        if obs is None:      # rows padded to 16 bytes so the kernel can store them with one TMA bulk copy (pad columns = 0)
            obs = torch.zeros((N, (self.obs_dim + 3) // 4 * 4), dtype=f32, device=dev)[:, :self.obs_dim]
        else:
            if not (torch.is_tensor(obs) and obs.is_cuda and obs.dtype == f32 and obs.dim() == 2 and obs.stride(1) == 1):
                obs = _req(obs, f32, "obs", dev)
            assert tuple(obs.shape) == (N, self.obs_dim), f"obs: shape {tuple(obs.shape)} != {(N, self.obs_dim)}"
        self.obs = obs
        self.rew = out(rew, (N,), f32, "rew")
        self.reward_raw = out(reward_raw, (N, rw), f32, "reward_raw")
        self.reset = out(reset, (N,), i64, "reset")
        self.terminate = out(terminate, (N,), i64, "terminate")
        S = cfg.amp_steps
        self.amp_obs_buf = out(amp_obs_buf, (N, S, self.amp_dim), f32, "amp_obs_buf") if with_amp else None
        if amp_hist_in is not None:
            amp_hist_in = _req(amp_hist_in, f32, "amp_hist_in", dev)
            assert amp_hist_in.shape == (N, S, self.amp_dim)
        elif with_amp and amp_shift and not amp_ring:
            amp_hist_in = self.amp_obs_buf             # in-place shift, the reference's semantics
        self.amp_ring = bool(amp_ring and with_amp)
        self.ring_head = 0
        self.ring_head_dev = None
        if ring_head_dev is not None:
            assert self.amp_ring and ring_head_dev.dtype == torch.int32 and ring_head_dev.is_cuda and ring_head_dev.numel() == 1
            self.ring_head_dev = ring_head_dev
            self.ring_head = None            # lives on the device only
        self.ref_body_pos = torch.zeros(N, J, 3, device=dev) if with_ref_buffers else None
        self.ref_body_rot = torch.zeros(N, J, 4, device=dev) if with_ref_buffers else None
        self.ref_body_vel = torch.zeros(N, J, 3, device=dev) if with_ref_buffers else None
        self.ref_body_ang_vel = torch.zeros(N, J, 3, device=dev) if with_ref_buffers else None

        # per-body termination threshold, +inf outside reset_bodies (compute_humanoid_im_reset is fed the subset)
        td = torch.as_tensor(cfg.term_dist, dtype=f32).expand(J).clone() if not torch.is_tensor(cfg.term_dist) else cfg.term_dist.float().cpu().clone()
        rb = list(range(J)) if cfg.reset_bodies is None else [int(b) for b in cfg.reset_bodies]
        thr = torch.full((J,), float("inf"))
        thr[rb] = td[rb]
        if J > _lib.PHC_MAX_BODIES or len(joints) > _lib.PHC_MAX_AMP_JOINTS:
            raise PhcError(f"phc_env_step supports at most {_lib.PHC_MAX_BODIES} bodies / {_lib.PHC_MAX_AMP_JOINTS} AMP joints")
        self._term_thresh = thr
        self._keep = dict(body_state=body_state, dof_state=dof_state, dof_force=dof_force,
                          progress=_req(progress, i64, "progress", dev), motion_ids=_req(motion_ids, i64, "motion_ids", dev),
                          start_times=_req(start_times, f32, "start_times", dev),
                          start_offsets=_req(start_offsets, f32, "start_offsets", dev),
                          global_offset=_req(global_offset, f32, "global_offset", dev),
                          cycle_counter=None if cycle_counter is None else _req(cycle_counter, torch.int32, "cycle_counter", dev),
                          amp_hist_in=amp_hist_in)
        k = self._keep
        a = _lib.PhcStepArgs()
        a.body_state, a.dof_state, a.dof_force, a.bodies_per_env = body_state.data_ptr(), dof_state.data_ptr(), _ptr(dof_force if cfg.power_reward else None), bpe
        a.progress, a.motion_ids = k["progress"].data_ptr(), k["motion_ids"].data_ptr()
        self._env_motion = torch.zeros(N, 4, dtype=torch.int32, device=dev)      # PhcEnvMotion records (16 B each)
        a.env_motion = self._env_motion.data_ptr()
        a.start_times, a.start_offsets, a.global_offset = k["start_times"].data_ptr(), k["start_offsets"].data_ptr(), k["global_offset"].data_ptr()
        a.cycle_counter = _ptr(k["cycle_counter"])
        # zero_out_far / cycle_motion state: _point_goal [N] (in/out) and the per-step uniform numbers for wrapping clips
        if cfg.zero_out_far:
            k["point_goal"] = _req(point_goal, f32, "point_goal", dev)
            assert k["point_goal"].shape == (N,)
            a.point_goal = k["point_goal"].data_ptr()
        if cfg.cycle_motion:
            k["cycle_phase"] = _req(cycle_phase, f32, "cycle_phase", dev)
            assert k["cycle_phase"].shape == (N,) and cycle_counter is not None
            a.cycle_phase = k["cycle_phase"].data_ptr()
        # flags.im_eval extras (humanoid_im.py:674-680): mpjpe [N] and the reference positions it is measured against [N, J, 3]
        self.mpjpe = torch.zeros(N, dtype=f32, device=dev) if with_eval_extras else None
        self.body_pos_gt = torch.zeros(N, J, 3, dtype=f32, device=dev) if with_eval_extras else None
        a.mpjpe, a.body_pos_gt = _ptr(self.mpjpe), _ptr(self.body_pos_gt)
        a.close_distance, a.far_distance, a.max_episode_length = cfg.close_distance, cfg.far_distance, int(cfg.max_episode_length)
        k["only_where"] = None if only_where is None else _req(only_where, i64, "only_where", dev)
        a.only_where = _ptr(k["only_where"])
        a.lib = mlib.c
        a.num_envs, a.time_steps, a.dt, a.traj_dt, a.flags = N, cfg.time_steps, cfg.dt, cfg.traj_dt, flags
        a.k_pos, a.k_rot, a.k_vel, a.k_ang_vel = cfg.k_pos, cfg.k_rot, cfg.k_vel, cfg.k_ang_vel
        a.w_pos, a.w_rot, a.w_vel, a.w_ang_vel = cfg.w_pos, cfg.w_rot, cfg.w_vel, cfg.w_ang_vel
        a.power_coef = cfg.power_coef
        for i in range(J):
            a.term_thresh[i] = float(thr[i])
        a.term_dist_mean = float(td[rb[0]])
        for i in range(E):
            a.ext_parent[i] = int(cfg.ext_parents[i])
            for c in range(3):
                a.ext_pos[i][c] = float(cfg.ext_pos[i][c])
        a.num_key_bodies = len(cfg.key_bodies)
        for i, b in enumerate(cfg.key_bodies):
            a.key_bodies[i] = int(b)
        for i, jt in enumerate(joints):
            a.amp_joints[i] = int(jt)
        a.num_amp_joints = len(joints)
        a.obs, a.obs_stride = self.obs.data_ptr(), self.obs.stride(0)
        a.rew, a.reward_raw, a.reset, a.terminate = self.rew.data_ptr(), self.reward_raw.data_ptr(), self.reset.data_ptr(), self.terminate.data_ptr()
        a.amp_out = _ptr(self.amp_obs_buf)
        a.amp_hist_in = _ptr(amp_hist_in) if with_amp else None
        a.amp_out_stride, a.amp_steps = S * self.amp_dim, S
        a.ref_body_pos, a.ref_body_rot = _ptr(self.ref_body_pos), _ptr(self.ref_body_rot)
        a.ref_body_vel, a.ref_body_ang_vel = _ptr(self.ref_body_vel), _ptr(self.ref_body_ang_vel)
        if ref_cache is not None:
            ref_cache = _req(ref_cache, f32, "ref_cache", dev)
            assert tuple(ref_cache.shape) == (N, int(mlib.frames_body.shape[1])), f"ref_cache: expected {(N, int(mlib.frames_body.shape[1]))}"
        self.ref_cache = ref_cache
        a.ref_cache = _ptr(ref_cache)
        a.ring_head = _ptr(self.ring_head_dev)
        if cfg.track_bodies is not None:
            tb = [int(b) for b in cfg.track_bodies]
            if len(set(tb)) != len(tb) or any(b < 0 or b >= J for b in tb):
                raise PhcError("EnvStepConfig.track_bodies: distinct body ids in [0, J)")
            a.num_track = len(tb)
            for b in range(_lib.PHC_MAX_BODIES):
                a.track_slot[b] = -1
            for pos, b in enumerate(tb):
                a.track_slot[b] = pos
        if occlusion is not None:
            if occlusion.dtype == torch.bool:
                occlusion = occlusion.view(torch.uint8)
            k["occlusion"] = _req(occlusion, torch.uint8, "occlusion", dev)
            assert tuple(occlusion.shape) == (N, K)
            a.occlusion = k["occlusion"].data_ptr()
        if shape_params is not None:
            k["shape_params"] = _req(shape_params, f32, "shape_params", dev)
            assert shape_params.shape[0] == N
            a.shape_params, a.num_shape = k["shape_params"].data_ptr(), ns
        if limb_weights is not None:
            k["limb_weights"] = _req(limb_weights, f32, "limb_weights", dev)
            assert limb_weights.shape[0] == N
            a.limb_weights, a.num_limb = k["limb_weights"].data_ptr(), nl
        self.args = a
        self._args_ref = C.byref(a)
        self.refresh_motion_params()

    def set_recovery_counter(self, counter: torch.Tensor) -> None:
        """Turn on the get-up schedule's recovery episodes (PHC_FLAG_RECOVERY): every later run() decrements `counter` (int32 [N],
        HumanoidImGetup._recovery_counter) and keeps envs with a running counter from resetting or advancing their progress."""
        self._keep["recovery_counter"] = _req(counter, torch.int32, "recovery_counter", self.device)
        assert counter.shape == (self.N,)
        self.args.recovery_counter = counter.data_ptr()
        self.args.flags |= _lib.PHC_FLAG_RECOVERY

    def set_motion_lib(self, mlib: PackedMotionLib) -> None:
        """Re-point the plan at a re-loaded motion library of the same character (HumanoidIm.resample_motions): new frame tables,
        new per-env motion records; every other pointer of the launch stays."""
        if mlib.num_bodies != self.mlib.num_bodies or mlib.num_ext_bodies != self.mlib.num_ext_bodies or mlib.dofs != self.mlib.dofs:
            raise PhcError("set_motion_lib: the new library must describe the same character (bodies / extend bodies / dofs)")
        self.mlib = mlib
        self.args.lib = mlib.c
        self.refresh_motion_params()

    def refresh_motion_params(self) -> None:
        """Re-gather the per-env motion parameters; call whenever `motion_ids` (HumanoidIm._sampled_motion_ids) changes."""
        _lib.check(self._lib.phc_env_motion_gather(C.byref(self.mlib.c), self._keep["motion_ids"].data_ptr(), self.N,
                                                   self._env_motion.data_ptr(), _stream()), "phc_env_motion_gather")

    def advance_ring(self) -> int:
        """Move the ring head one slot back (the slot that will receive this step's AMP vector) and re-point amp_out."""
        S = self.cfg.amp_steps
        if self.ring_head_dev is not None:
            _lib.check(self._lib.phc_ring_advance(self.ring_head_dev.data_ptr(), S, _stream()), "phc_ring_advance")
            return -1
        self.ring_head = (self.ring_head - 1) % S
        self.args.amp_out = self.amp_obs_buf.data_ptr() + self.ring_head * self.amp_dim * 4
        return self.ring_head

    def run(self, stream: Optional[int] = None) -> None:
        rc = self._lib.phc_env_step(self._args_ref, _stream() if stream is None else stream)
        if rc:
            _lib.check(rc, "phc_env_step")


def amp_obs_demo(mlib: PackedMotionLib, cfg: EnvStepConfig, motion_ids: torch.Tensor, times0: torch.Tensor,
                 first_step: int = 0, num_steps: Optional[int] = None, out: Optional[torch.Tensor] = None,
                 only_where: Optional[torch.Tensor] = None, slot_offset: int = 0, slot_offset_dev: Optional[torch.Tensor] = None) -> torch.Tensor:
    """build_amp_obs_demo (humanoid_amp.py:253-284; first_step=0) / _init_amp_obs_ref (:575-603; first_step=1)."""
    lib = _lib.load()
    dev = mlib.device
    ids = _req(motion_ids, torch.int64, "motion_ids", dev)
    t0 = _req(times0, torch.float32, "times0", dev)
    n = int(ids.shape[0])
    S = cfg.amp_steps if num_steps is None else num_steps
    robot = mlib.num_dofs > 0
    joints = [] if robot else cfg.amp_joint_list(mlib.num_bodies)
    A = (lib.phc_amp_obs_dim_robot(mlib.num_dofs, len(cfg.key_bodies), cfg.flags()) if robot
         else lib.phc_amp_obs_dim(len(joints), len(cfg.key_bodies), cfg.flags()))
    if out is None:
        out = torch.empty(n, S, A, dtype=torch.float32, device=dev)
    else:
        out = _req(out, torch.float32, "out", dev)
        assert out.shape[0] == n and out.shape[-1] == A and out.stride(0) >= S * A
    kb = (C.c_int32 * len(cfg.key_bodies))(*[int(b) for b in cfg.key_bodies])
    aj = (C.c_int32 * max(1, len(joints)))(*[int(j) for j in joints])
    with torch.cuda.device(dev):
        _lib.check(lib.phc_amp_obs_demo_ring(C.byref(mlib.c), ids.data_ptr(), t0.data_ptr(), n, first_step, S, cfg.dt,
                                             cfg.flags(), C.cast(kb, C.c_void_p), len(cfg.key_bodies), C.cast(aj, C.c_void_p),
                                             len(joints), out.data_ptr(), out.stride(0),
                                             None if only_where is None else _req(only_where, torch.int64, "only_where", dev).data_ptr(),
                                             int(slot_offset), _ptr(slot_offset_dev), _stream()), "phc_amp_obs_demo")
    return out


def getup_reset(mask: torch.Tensor, terminate_in: torch.Tensor, u_rec: torch.Tensor, u_fall: torch.Tensor, perm: torch.Tensor,
                p_rec: torch.Tensor, p_fall: torch.Tensor, recovery_steps: int, fall_root: torch.Tensor, fall_dof_pos: torch.Tensor,
                available: torch.Tensor, assignment: torch.Tensor, recovery_counter: torch.Tensor, body_state: torch.Tensor,
                dof_state: torch.Tensor, progress: torch.Tensor, reset: torch.Tensor, terminate: torch.Tensor, ref_init: torch.Tensor,
                fall: torch.Tensor) -> None:
    """phc_getup_reset: the reset selection of HumanoidImGetup._reset_actors (humanoid_im_getup.py:135-182) for the envs with mask != 0.
    Writes ref_init / fall (int64 0/1 masks), the fall envs' root record and dof state, the bank marks, assignments and counters."""
    lib = _lib.load()
    dev = body_state.device
    i64, f32 = torch.int64, torch.float32
    n = int(mask.shape[0])
    D = int(dof_state.shape[1])
    for t, dt, name in ((mask, i64, "mask"), (terminate_in, i64, "terminate_in"), (u_rec, f32, "u_rec"), (u_fall, f32, "u_fall"),
                        (perm, i64, "perm"), (p_rec, f32, "p_rec"), (p_fall, f32, "p_fall"), (fall_root, f32, "fall_root"),
                        (fall_dof_pos, f32, "fall_dof_pos"), (available, i64, "available"), (assignment, i64, "assignment"),
                        (recovery_counter, torch.int32, "recovery_counter"), (body_state, f32, "body_state"), (dof_state, f32, "dof_state"),
                        (progress, i64, "progress"), (reset, i64, "reset"), (terminate, i64, "terminate"), (ref_init, i64, "ref_init"),
                        (fall, i64, "fall")):
        _req(t, dt, name, dev)
    P = int(fall_root.shape[0])
    assert fall_root.shape == (P, 13) and fall_dof_pos.shape == (P, D) and perm.shape == (P,) and available.shape == (P,)
    assert body_state.shape[0] == n and dof_state.shape == (n, D, 2)
    for t in (terminate_in, u_rec, u_fall, assignment, recovery_counter, progress, reset, terminate, ref_init, fall):
        assert t.shape == (n,)
    _lib.check(lib.phc_getup_reset(mask.data_ptr(), terminate_in.data_ptr(), u_rec.data_ptr(), u_fall.data_ptr(), perm.data_ptr(),
                                   p_rec.data_ptr(), p_fall.data_ptr(), int(recovery_steps), fall_root.data_ptr(), fall_dof_pos.data_ptr(), P,
                                   available.data_ptr(), assignment.data_ptr(), recovery_counter.data_ptr(), n, body_state.data_ptr(),
                                   int(body_state.shape[1]), dof_state.data_ptr(), D, progress.data_ptr(), reset.data_ptr(),
                                   terminate.data_ptr(), ref_init.data_ptr(), fall.data_ptr(), _stream()), "phc_getup_reset")


def amp_ring_fill(ring: torch.Tensor, head, mask: torch.Tensor) -> None:
    """phc_amp_ring_fill: every slot of the masked envs' AMP rows = the newest slot (`head`: the int32 [1] device ring head, or None
    for a newest-first window whose newest slot is 0) -- _init_amp_obs_default (humanoid_amp.py:570-573)."""
    lib = _lib.load()
    n, S, A = ring.shape
    _req(ring, torch.float32, "ring")
    _req(mask, torch.int64, "mask", ring.device)
    _lib.check(lib.phc_amp_ring_fill(ring.data_ptr(), ring.stride(0), n, S, A, _ptr(head), mask.data_ptr(), _stream()), "phc_amp_ring_fill")


def eval_metrics_step(body_pos: torch.Tensor, body_pos_gt: torch.Tensor, num_steps: torch.Tensor, t: int, ring: torch.Tensor,
                      acc: torch.Tensor) -> None:
    """phc_eval_metrics_step: adds eval step `t`'s frame to the per-env metric sums `acc` [N, 8] fp64 (mpjpe_g, mpjpe_l, mpjpe_pa,
    vel_dist, accel_dist in metres, then three frame counts) -- the per-step part of compute_metrics_lite over the reference's clip
    slices (im_amp.py:244-363).  body_pos: [N, J, 3] fp32, any env / body strides with x, y, z contiguous (the `[..., :J, 0:3]` view
    of the rigid-body state); body_pos_gt [N, J, 3]; num_steps [N] int32; ring [2, N, J, 3] fp32 (d_{t-1}, d_{t-2})."""
    if body_pos.dim() != 3 or body_pos.shape[-1] != 3:
        raise ValueError(f"body_pos: expected [N, J, 3], got {tuple(body_pos.shape)}")
    n, J = int(body_pos.shape[0]), int(body_pos.shape[1])
    if not 1 <= J <= 64:
        raise ValueError(f"eval_metrics_step: J = {J} bodies, the kernel takes 1..64")
    if not body_pos.is_cuda:
        raise PhcError(f"body_pos: phc_b200 runs on CUDA tensors only (got {body_pos.device}); there is no CPU fallback")
    if body_pos.dtype != torch.float32 or body_pos.stride(-1) != 1:
        raise ValueError("body_pos: fp32 with x, y, z contiguous")
    dev = body_pos.device
    _req(body_pos_gt, torch.float32, "body_pos_gt", dev)
    _req(num_steps, torch.int32, "num_steps", dev)
    _req(ring, torch.float32, "ring", dev)
    _req(acc, torch.float64, "acc", dev)
    assert body_pos_gt.shape == (n, J, 3) and num_steps.shape == (n,) and ring.shape == (2, n, J, 3)
    assert acc.shape == (n, _lib.PHC_EVAL_ACC_FIELDS)
    lib = _lib.load()
    _lib.check(lib.phc_eval_metrics_step(body_pos.data_ptr(), body_pos.stride(0), body_pos.stride(1), body_pos.stride(2),
                                         body_pos_gt.data_ptr(), num_steps.data_ptr(), int(t), n, J, ring.data_ptr(), acc.data_ptr(),
                                         _stream()), "phc_eval_metrics_step")


def episode_stats(rewards: torch.Tensor, dones: torch.Tensor, cur_r: torch.Tensor, cur_l: torch.Tensor, meter_mean: torch.Tensor,
                  meter_size: torch.Tensor, games_to_track: int) -> None:
    """phc_episode_stats: one rollout step of the episode bookkeeping (amp_agent.py:358-369).  cur_r += rewards and cur_l += 1, the
    returns and lengths of the envs with dones != 0 are folded into the meters (rl_games' AverageMeter.update, max_size =
    games_to_track), then both are zeroed where done.  rewards, cur_r, cur_l [N] fp32; dones [N] int64 (reset_buf);
    meter_mean [2] fp32 and meter_size [2] int32: game_rewards, game_lengths."""
    dev = cur_r.device
    _req(rewards, torch.float32, "rewards", dev)
    _req(dones, torch.int64, "dones", dev)
    _req(cur_r, torch.float32, "cur_r", dev)
    _req(cur_l, torch.float32, "cur_l", dev)
    _req(meter_mean, torch.float32, "meter_mean", dev)
    _req(meter_size, torch.int32, "meter_size", dev)
    n = cur_r.numel()
    if rewards.numel() != n or dones.numel() != n or cur_l.numel() != n or meter_mean.numel() != 2 or meter_size.numel() != 2:
        raise ValueError("episode_stats: rewards, dones, cur_r, cur_l must have N elements, meter_mean and meter_size 2")
    lib = _lib.load()
    _lib.check(lib.phc_episode_stats(rewards.data_ptr(), dones.data_ptr(), n, cur_r.data_ptr(), cur_l.data_ptr(), meter_mean.data_ptr(),
                                     meter_size.data_ptr(), int(games_to_track), _stream()), "phc_episode_stats")


def amp_window_export(ring: torch.Tensor, head, out: torch.Tensor) -> torch.Tensor:
    """out[n, k, :] = ring[n, (head + k) % S, :] -- newest-first AMP window from the ring (phc_amp_window_export).
    `head`: an int, or the int32 [1] device tensor that holds it."""
    lib = _lib.load()
    n, S, A = ring.shape
    _req(ring, torch.float32, "ring")
    assert out.dtype == torch.float32 and out.is_cuda and out.shape[0] == n and out.stride(-1) == 1 and out.numel() == n * S * A
    dev_head = head if torch.is_tensor(head) else None
    _lib.check(lib.phc_amp_window_export_ring(ring.data_ptr(), ring.stride(0), n, S, A, 0 if dev_head is not None else int(head), _ptr(dev_head),
                                              out.data_ptr(), out.stride(0), _stream()), "phc_amp_window_export")
    return out


# ------------------------------------------------------------------------------------------------------------
# PPO scalars
# ------------------------------------------------------------------------------------------------------------
def gae(fdones: torch.Tensor, values: torch.Tensor, rewards: torch.Tensor, next_values: torch.Tensor, gamma: float,
        tau: float, want_returns: bool = True):
    """CommonAgent.discount_values (+ returns).  Time-major [T,N] or [T,N,1] fp32 tensors."""
    lib = _lib.load()
    dev = rewards.device
    shape = rewards.shape
    T, N = int(shape[0]), int(shape[1])
    fd = _req(fdones, torch.float32, "fdones", dev)
    v, r, nv = _req(values, torch.float32, "values", dev), _req(rewards, torch.float32, "rewards", dev), _req(next_values, torch.float32, "next_values", dev)
    assert fd.numel() == v.numel() == r.numel() == nv.numel() == T * N
    advs = torch.empty(shape, dtype=torch.float32, device=dev)
    rets = torch.empty(shape, dtype=torch.float32, device=dev) if want_returns else None
    with torch.cuda.device(dev):
        _lib.check(lib.phc_gae(fd.data_ptr(), v.data_ptr(), r.data_ptr(), nv.data_ptr(), T, N, gamma, tau,
                               advs.data_ptr(), _ptr(rets), _stream()), "phc_gae")
    return (advs, rets) if want_returns else advs


def adv_norm(returns: torch.Tensor, values: torch.Tensor, normalize: bool = True) -> torch.Tensor:
    """CommonAgent._calc_advs: [B,1] (or [B]) returns / values -> normalised advantages [B]."""
    lib = _lib.load()
    dev = returns.device
    r, v = _req(returns, torch.float32, "returns", dev), _req(values, torch.float32, "values", dev)
    n = r.numel()
    assert v.numel() == n
    advs = torch.empty(n, dtype=torch.float32, device=dev)
    ws = torch.empty(max(1, lib.phc_adv_norm_workspace_bytes(n) // 8), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.phc_adv_norm(r.data_ptr(), v.data_ptr(), n, 1 if normalize else 0, advs.data_ptr(),
                                    ws.data_ptr(), _stream()), "phc_adv_norm")
    return advs
