"""Generate tests/golden/getup_sched.npz: the get-up schedule of the UNMODIFIED reference (phc/env/tasks/humanoid_im_getup.py).

Like make_golden_kp.py it builds the environment with make_golden.build_ref_env (an `object.__new__` instance with every attribute
set by hand, imported through ref_shim) and re-classes it as the reference's HumanoidImGetup, so the reference's own methods run.
The inputs of the step cases are those of getup.npz / getup_smplx.npz, read from there rather than stored again.

  step24, step52   three consecutive env steps (env_im_getup_mcp.yaml: zero_out_far + cycle_motion, max_episode_length 15) with
                   recovery counters 0..5: _update_recovery_count + _update_cycle_count (pre_physics_step, :76-80 and
                   humanoid_im.py:1076-1079), progress + 1, HumanoidImGetup._compute_reset over HumanoidIm's (clip wrap-around and
                   pass_time included, :203-210), observations, AMP.  Counters run down to 0, early termination is on.
  sel24, sel52     four consecutive resets of a persistent fall-state bank: two before getup_udpate_epoch (p_rec 0, p_fall 1) and two
                   after (0.5, 0.3), random reset masks and terminations.  HumanoidImGetup._reset_actors (:135-182) runs as shipped;
                   only HumanoidIm._reset_actors (the reference-state init, pinned by reset.npz) is replaced by a recorder.  Then
                   _reset_env_tensors' counters (humanoid.py:615-617), _compute_observations(env_ids) and HumanoidImGetup._init_amp_obs
                   with the reference-state part left out (recovery envs: newest slot; fall envs: every slot, humanoid_amp.py:559-573).
The generator, and only the generator, wraps torch.bernoulli and torch.randperm to record the draws the reference consumed: per env
uniforms u_rec / u_fall (bernoulli(p) == 1 <=> u < p) and the bank permutation (available_ids[randperm(n)] followed by the taken
states), which the device kernel then gets as inputs.

  python tests/golden/make_golden_getup_sched.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import build_ref_env, save, syn  # noqa: E402  (imports the reference through its shim)

STEPS = 3
RESETS = ((0.0, 1.0), (0.0, 1.0), (0.5, 0.3), (0.5, 0.3))


def source(name):
    z = np.load(os.path.join(HERE, name))
    g = {k: torch.from_numpy(z[k]) for k in z.files}
    m = syn.MotionData(**{k: g["tab_" + k] for k in syn.MotionData.__dataclass_fields__})
    st = syn.EnvState(**{k: g["in_" + k].clone() for k in syn.EnvState.__dataclass_fields__})
    return g, m, st


def getup_env(m, st, J):
    from phc.env.tasks.humanoid_im_getup import HumanoidImGetup
    env = build_ref_env(m, st)
    if J != 24:          # SMPL-X shapes, set up as make_golden.gen_smplx
        env.humanoid_type = "smplx"
        env._reset_bodies_id = torch.arange(J)
        env._key_body_ids = torch.tensor(syn.SMPLX_KEY_BODIES)
        env.dof_subset, env._has_dof_subset = torch.tensor([]).long(), False
        env._dof_names = [f"j{i}" for i in range(1, J)]
    env.__class__ = HumanoidImGetup
    env.zero_out_far, env.zero_out_far_train, env.cycle_motion, env.cycle_motion_xp = True, False, True, False
    env.close_distance, env.far_distance = 0.25, 3
    env.max_episode_length = 15
    env._humanoid_root_states = env._rigid_body_state_reshaped[:, 0, :]
    env._motion_lib._device = torch.device("cpu")
    env._recovery_steps = 90
    return env


def gen_step(d, tag, src, J):
    g, m, st = source(src)
    N = st.body_state.shape[0]
    env = getup_env(m, st, J)
    gen = torch.Generator().manual_seed(31 + J)
    rc_in = torch.tensor([0, 0, 1, 2, 3, 5], dtype=torch.int)[torch.randint(0, 6, (N,), generator=gen)]
    env._recovery_counter = rc_in.clone()
    env._cycle_counter = g["in_cycle_counter"].clone()
    env._point_goal = g["in_point_goal"].clone()
    d[f"{tag}_in_recovery_counter"] = rc_in
    for k in range(STEPS):
        env._update_recovery_count()                         # pre_physics_step (humanoid_im_getup.py:76-80)
        env._update_cycle_count()
        if k > 0:
            env.progress_buf += 1                            # the step inputs already hold the incremented progress
        t_now = env.progress_buf * env.dt + env._motion_start_times + env._motion_start_times_offset
        wrap = t_now >= m.lengths[env._sampled_motion_ids]
        torch.manual_seed(77 + k)                            # the numbers sample_time_interval draws for the wrapping envs
        phase = torch.zeros(N)
        phase[wrap] = torch.rand(int(wrap.sum()))
        env._compute_reward(None)
        torch.manual_seed(77 + k)
        env._compute_reset()
        env._compute_observations()
        S = env._num_amp_obs_steps
        env._hist_amp_obs_buf[:] = env._amp_obs_buf[:, 0:(S - 1)].clone()      # make_golden.run_ref_step explains the fallback
        env._compute_amp_observations()
        p = f"{tag}_{k}_"
        d[p + "in_cycle_phase"] = phase
        # the observation rows of the envs still recovering (the others are getup.npz's kind of row) and no AMP window (the recovery
        # counter does not enter it): keeps the file small
        rows = (env._recovery_counter > 0).nonzero().squeeze(-1)
        d[p + "out_obs_rows"], d[p + "out_obs"] = rows, env.obs_buf[rows].clone()
        for name, v in (("rew", env.rew_buf), ("reward_raw", env.reward_raw), ("reset", env.reset_buf),
                        ("terminate", env._terminate_buf), ("progress", env.progress_buf), ("recovery_counter", env._recovery_counter),
                        ("cycle_counter", env._cycle_counter), ("start_times", env._motion_start_times),
                        ("start_offsets", env._motion_start_times_offset), ("global_offset", env._global_offset),
                        ("point_goal", env._point_goal)):
            d[p + "out_" + name] = v.clone()
        print(f"{tag} step {k}: recovering {int((env._recovery_counter > 0).sum())}, wrapping {int(wrap.sum())}, "
              f"resets {int(env.reset_buf.sum())}, terminated {int(env._terminate_buf.sum())}")


def gen_select(d, tag, src, J):
    from phc.env.tasks import humanoid_im as him
    from phc.env.tasks.humanoid_im_getup import HumanoidImGetup
    g, m, st = source(src)
    N, D = st.body_state.shape[0], st.dof_state.shape[1]
    env = getup_env(m, st, J)
    gen = torch.Generator().manual_seed(57 + J)
    env._recovery_counter = torch.zeros(N, dtype=torch.int)
    env._point_goal = torch.zeros(N)
    env.availalbe_fall_states = torch.zeros(N).long()
    env.fall_id_assignments = torch.zeros(N).long()
    # the fall-state bank (_generate_fall_states, :82-125, needs the simulator): root states with random unit rotations, zero velocity
    fall_root = torch.randn(N, 13, generator=gen)
    fall_root[:, 3:7] = torch.nn.functional.normalize(fall_root[:, 3:7], dim=-1)
    fall_root[:, 7:13] = 0
    env._fall_root_states = fall_root
    env._fall_dof_pos = torch.randn(N, D, generator=gen) * 0.3
    env._fall_dof_vel = torch.zeros(N, D)
    d[f"{tag}_fall_root"], d[f"{tag}_fall_dof_pos"] = fall_root, env._fall_dof_pos
    real_bern, real_perm, real_ref_reset = torch.bernoulli, torch.randperm, him.HumanoidIm._reset_actors
    draws = {}

    def bern(p, *a, **k):
        u = torch.rand(p.shape, generator=gen)
        draws.setdefault("u", []).append(u)
        return (u < p.float()).to(p.dtype)

    def perm(n, *a, **k):
        r = real_perm(n, generator=gen)
        draws["perm"] = (r, (env.availalbe_fall_states == 0).nonzero().squeeze(-1))
        return r

    def ref_init_recorder(self, env_ids):             # HumanoidIm._reset_actors: the reference-state init, pinned by reset.npz
        draws["ref_init"] = env_ids.clone()
        self._reset_default_env_ids, self._reset_ref_env_ids = [], []

    torch.bernoulli, torch.randperm, him.HumanoidIm._reset_actors = bern, perm, ref_init_recorder
    stale_total = 0
    try:
        for r, (p_rec, p_fall) in enumerate(RESETS):
            draws.clear()
            mask = torch.rand(N, generator=gen) < 0.5
            term = (torch.rand(N, generator=gen) < 0.5).long()
            env._terminate_buf = term.clone()
            env.progress_buf = torch.randint(1, 15, (N,), generator=gen)
            env.reset_buf = (torch.rand(N, generator=gen) < 0.5).long()
            env._recovery_episode_prob, env._fall_init_prob = p_rec, p_fall
            p = f"{tag}_{r}_"
            # inputs: the draws below and these; the simulator state, bank marks, assignments, counters and AMP windows carry over from
            # the previous reset (the first one starts from the source golden's inputs and a zero bank state)
            for name, v in (("mask", mask.long()), ("terminate", term), ("progress", env.progress_buf), ("reset", env.reset_buf)):
                d[p + "in_" + name] = v.clone()
            env_ids = mask.nonzero().squeeze(-1)
            held = env.availalbe_fall_states.clone()
            stale_total += int(sum(1 for e in env_ids.tolist() if held[env.fall_id_assignments[e]] == 1 and
                                   (env.fall_id_assignments == env.fall_id_assignments[e]).sum() > 1))
            env._reset_fall_env_ids = []                                                 # HumanoidImGetup._reset_envs (:184-188)
            env._reset_default_env_ids, env._reset_ref_env_ids = [], []                  # HumanoidAMP._reset_envs (humanoid_amp.py:378-387)
            HumanoidImGetup._reset_actors(env, env_ids)                                  # :135-182 as shipped
            env.progress_buf[env_ids] = 0                                                # _reset_env_tensors (humanoid.py:615-617)
            env.reset_buf[env_ids] = 0
            env._terminate_buf[env_ids] = 0
            env._compute_observations(env_ids)
            HumanoidImGetup._init_amp_obs(env, env_ids)                                  # :190-196 (reference-state part recorded away)
            # the draws as the kernel takes them
            u = draws.get("u", [])
            u_rec, u_fall = torch.ones(N), torch.ones(N)
            u_rec[env_ids] = u[0]
            rec = (u[0] < p_rec) & (term[env_ids] == 1)
            u_fall[env_ids[~rec]] = u[1]
            if "perm" in draws:
                rp, avail_ids = draws["perm"]
                first = avail_ids[rp]
                rest = torch.tensor([s for s in range(N) if s not in set(first.tolist())], dtype=torch.long)
                bank_perm = torch.cat([first, rest])
            else:
                bank_perm = torch.arange(N)
            ref_ids = draws.get("ref_init", torch.zeros(0, dtype=torch.long))
            fall_ids = env._reset_fall_env_ids if len(env._reset_fall_env_ids) else torch.zeros(0, dtype=torch.long)
            ref_mask, fall_mask = torch.zeros(N, dtype=torch.long), torch.zeros(N, dtype=torch.long)
            ref_mask[ref_ids], fall_mask[fall_ids] = 1, 1
            d[p + "in_u_rec"], d[p + "in_u_fall"], d[p + "in_perm"] = u_rec, u_fall, bank_perm
            d[p + "in_probs"] = torch.tensor([p_rec, p_fall], dtype=torch.float32)
            for name, v in (("available", env.availalbe_fall_states), ("assignment", env.fall_id_assignments),
                            ("recovery_counter", env._recovery_counter), ("progress", env.progress_buf), ("reset", env.reset_buf),
                            ("terminate", env._terminate_buf), ("root_state", env._rigid_body_state_reshaped[:, 0]),
                            ("dof_pos", env._dof_pos), ("ref_init", ref_mask), ("fall", fall_mask)):
                d[p + "out_" + name] = v.clone()
            # observation rows and newest AMP slot of the fall and recovery envs (fall envs: every slot equal, checked by the tests), for
            # the first reset of each schedule phase: keeps the file small
            rows = ((fall_mask == 1) | (mask & (ref_mask == 0))).nonzero().squeeze(-1)
            d[p + "out_rows"] = rows
            d[p + "out_amp_newest"] = env._amp_obs_buf[rows, 0].clone()
            assert torch.equal(env._amp_obs_buf[fall_ids], env._amp_obs_buf[fall_ids, :1].expand_as(env._amp_obs_buf[fall_ids]))
            if r in (0, 2):
                d[p + "out_obs"] = env.obs_buf[rows].clone()
            print(f"{tag} reset {r} (p_rec {p_rec}, p_fall {p_fall}): resetting {len(env_ids)}, recovery {int(rec.sum())}, "
                  f"fall {int(fall_mask.sum())}, ref-init {int(ref_mask.sum())}")
    finally:
        torch.bernoulli, torch.randperm, him.HumanoidIm._reset_actors = real_bern, real_perm, real_ref_reset
    print(f"{tag}: resetting envs whose stale assignment freed a state another env holds: {stale_total}")


def main():
    d = {}
    gen_step(d, "step24", "getup.npz", 24)
    gen_step(d, "step52", "getup_smplx.npz", 52)
    gen_select(d, "sel24", "getup.npz", 24)
    gen_select(d, "sel52", "getup_smplx.npz", 52)
    save("getup_sched.npz", d)


if __name__ == "__main__":
    main()
