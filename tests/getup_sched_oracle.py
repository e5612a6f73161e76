"""The get-up schedule of HumanoidImGetup (phc/env/tasks/humanoid_im_getup.py) restated in plain torch, statement for statement, with
the random draws made explicit: `torch.bernoulli(p) == 1` is `u < p` for a caller-supplied uniform u, and `available_ids[randperm(n)]` is
the available states taken in the order of a caller-supplied permutation of the bank.  Test infrastructure; the existing oracle is
untouched.

  reset_select : _reset_actors (:135-182) + _reset_env_tensors' progress / reset / terminate clear (humanoid.py:615-617)
  recovery_step: _update_recovery_count (:198-201) + the _compute_reset override (:203-210) applied to what a plain step produced
"""
import torch


def reset_select(mask, terminate, u_rec, u_fall, perm, p_rec, p_fall, recovery_steps, fall_root, fall_dof_pos, available, assignment,
                 counter, body_state, dof_state, progress, reset, term):
    """In-place on clones of every mutable argument; returns dict of the results plus the ref-init and fall masks (int64 0/1)."""
    available, assignment, counter = available.clone(), assignment.clone(), counter.clone()
    body_state, dof_state, progress, reset, term = body_state.clone(), dof_state.clone(), progress.clone(), reset.clone(), term.clone()
    N = mask.shape[0]
    env_ids = mask.nonzero().flatten()
    available[assignment[env_ids]] = 0                                       # :136
    recovery_mask = (u_rec[env_ids] < p_rec) & (terminate[env_ids] == 1)     # :138-141
    recovery_ids = env_ids[recovery_mask]
    counter[recovery_ids] = recovery_steps                                   # :164-166
    nonrecovery_ids = env_ids[~recovery_mask]
    fall_mask = u_fall[nonrecovery_ids] < p_fall                             # :150-151
    fall_ids = nonrecovery_ids[fall_mask]
    if len(fall_ids) > 0:                                                    # _reset_fall_episode (:168-182)
        available[assignment[fall_ids]] = 0
        free_in_perm_order = perm[available[perm] == 0]
        assert free_in_perm_order.shape[0] >= fall_ids.shape[0]
        states = free_in_perm_order[:fall_ids.shape[0]]
        body_state[fall_ids, 0] = fall_root[states]
        dof_state[fall_ids, :, 0] = fall_dof_pos[states]
        dof_state[fall_ids, :, 1] = 0
        counter[fall_ids] = recovery_steps
        available[states] = 1
        assignment[fall_ids] = states
    nonfall_ids = nonrecovery_ids[~fall_mask]
    counter[nonfall_ids] = 0                                                 # :157-160
    for ids in (recovery_ids, fall_ids):
        progress[ids] = 0
        reset[ids] = 0
        term[ids] = 0
    ref_init = torch.zeros(N, dtype=torch.int64)
    ref_init[nonfall_ids] = 1
    fall = torch.zeros(N, dtype=torch.int64)
    fall[fall_ids] = 1
    return dict(available=available, assignment=assignment, counter=counter, body_state=body_state, dof_state=dof_state, progress=progress,
                reset=reset, terminate=term, ref_init=ref_init, fall=fall)


def recovery_step(counter, progress, reset, term):
    """counter: before the step; progress: the incremented progress the step ran with; reset / term: what the step without the
    override produced.  Returns (counter, progress, reset, terminate, recovering mask) after the override."""
    c = torch.clamp_min(counter - 1, 0)
    rec = c > 0
    return c, torch.where(rec, progress - 1, progress), torch.where(rec, torch.zeros_like(reset), reset), \
        torch.where(rec, torch.zeros_like(term), term), rec


def env_step_recovery(tab, cfg, body_state, dof_state, dof_force, progress, motion_ids, start_times, start_offsets, global_offset,
                      amp_hist, point_goal, cycle_counter, cycle_phase, recovery_counter, max_episode_length):
    """One step of HumanoidImGetup in the env_im_getup_mcp.yaml configuration on top of the existing oracle's getup step
    (oracle.phc_oracle.env_step_getup): reward, reset and the clip wrap-around at `progress`, then the recovery override, and for the
    envs still recovering the observation of `progress - 1` (humanoid.py:1634-1647) with the bookkeeping the wrap-around left
    (offset -progress*dt: the decremented observation time lands exactly on the re-based start).  Counters are the values before
    pre_physics_step's decrements.  Returns the oracle dict with `progress` and `recovery_counter` added."""
    from oracle import phc_oracle as O
    kw = dict(zero_out_far=True, cycle_motion=True, max_episode_length=max_episode_length)
    a = O.env_step_getup(tab, cfg, body_state, dof_state, dof_force, progress, motion_ids, start_times, start_offsets, global_offset,
                         amp_hist, point_goal, cycle_counter, cycle_phase, **kw)
    rc, prog, reset, term, rec = recovery_step(recovery_counter, progress, a["reset"], a["terminate"])
    b = O.env_step_getup(tab, cfg, body_state, dof_state, dof_force, prog, motion_ids, a["start_times"], a["start_offsets"],
                         a["global_offset"], amp_hist, point_goal, a["cycle_counter"] + 1, torch.zeros_like(cycle_phase), **kw)
    out = dict(a)
    out.update(reset=reset, terminate=term, progress=prog, recovery_counter=rc)
    out["obs"] = torch.where(rec[:, None], b["obs"], a["obs"])
    out["point_goal"] = torch.where(rec, b["point_goal"], a["point_goal"])
    return out
