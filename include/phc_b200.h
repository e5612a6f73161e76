/* phc_b200 -- C ABI of the GPU-native PHC hot path (libphc_b200.so, built for the H100: sm_90a).
 *
 * The reference (ZhengyiLuo/PHC) has NO native boundary: the whole path is Python/TorchScript.  This header is
 * where one is cut.  Every entry point replaces a group of reference functions (cited file:line, relative to the
 * reference checkout) and takes plain device pointers + sizes + a CUDA stream -- no torch types.  Ownership never
 * transfers: every buffer is allocated by the caller (a torch tensor in the Python host), the library allocates
 * nothing except the workspace objects created by the *_create calls below.
 *
 * All functions return 0 (PHC_OK) or a negative PHC_ERR_* code, never throw, never synchronise the device unless
 * documented.  `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Quaternions are xyzw fp32.
 */
#ifndef PHC_B200_H_
#define PHC_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Exported entry points (the library is built with -fvisibility=hidden). */
#if defined(_WIN32)
#define PHC_API __declspec(dllexport)
#else
#define PHC_API __attribute__((visibility("default")))
#endif

#define PHC_OK 0
#define PHC_ERR_INVALID_ARG (-1)  /* NULL pointer / bad size / misaligned table                          */
#define PHC_ERR_UNSUPPORTED (-2)  /* configuration outside what the kernels implement (see message)      */
#define PHC_ERR_CUDA (-3)         /* a CUDA runtime call failed; phc_last_error() has the cudaError text */

/* Library / build information.  phc_version() = 10000*major + 100*minor + patch. */
PHC_API int phc_version(void);
/* Thread-local, NUL-terminated description of the last non-zero return on this thread. */
PHC_API const char* phc_last_error(void);
/* Number of CUDA kernels this library has launched in the calling process (monotonic; bench.py reports the delta). */
PHC_API int64_t phc_launch_count(void);
/* SM architecture the library was compiled for (90 for sm_90a). */
PHC_API int phc_compiled_sm(void);

/* ------------------------------------------------------------------------------------------------------------
 * Motion library, packed device format
 *   replaces the table set MotionLibBase builds at load time: gts/grs/lrs/gvs/gavs/dvs
 *   (phc/utils/motion_lib_base.py:300-307).  One frame = one 16-byte aligned record so a frame bracket is two
 *   TMA bulk copies:  body record  [J][13] = pos3 rot4 vel3 angvel3  (the simulator's rigid-body layout,
 *   phc/env/tasks/humanoid.py:219-226), padded to body_stride floats (multiple of 4);
 *   joint record [J][4] local rotation then [J-1][3] dof velocity, padded to joint_stride floats.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct PhcMotionLib {
  const float* frames_body;         /* [num_frames_total, body_stride]                                       */
  const float* frames_joint;        /* [num_frames_total, joint_stride] or NULL (dof_pos/dof_vel unavailable) */
  const float* motion_len;          /* [num_motions] seconds          (_motion_lengths)                       */
  const float* motion_dt;           /* [num_motions] seconds / frame  (_motion_dt)                            */
  const int64_t* motion_num_frames; /* [num_motions]                  (_motion_num_frames)                    */
  const int64_t* length_starts;     /* [num_motions] first table row  (length_starts)                         */
  int64_t num_frames_total;
  int32_t num_motions;
  int32_t num_bodies;   /* J */
  int32_t body_stride;  /* floats per body record  = round_up(13*(J+E), 4)       */
  int32_t joint_stride; /* floats per joint record = round_up(4*J + 3*(J-1), 4), or round_up(2*D, 4) for hinge-joint robots */
  /* Robots (humanoid_type h1 / g1: phc/utils/motion_lib_real.py:236-361, humanoid_im.py:74-82, :916-923).  Zero for SMPL. */
  int32_t num_ext_bodies; /* E: "extend" bodies (head, hands ...) carried as records J..J+E-1 of every frame (the *_t tables);
                             they enter the tracking reward only                                                        */
  int32_t num_dofs;       /* D > 0: every joint is one hinge dof; the joint record is [dof_pos[D] | dof_vel[D]] and dof_pos is
                             interpolated linearly (motion_lib_real.py:283-285); 0: SMPL, D = 3(J-1) via local rotations   */
} PhcMotionLib;

/* Per-env copy of the motion parameters the step needs, gathered once by phc_env_motion_gather whenever motion_ids change
 * (HumanoidIm re-samples clips every `shape_resampling_interval` epochs, amp_agent.py:509-515): one 16-byte load per env
 * instead of motion_ids -> 4 dependent table look-ups on the per-step critical path. */
typedef struct PhcEnvMotion {
  float len;         /* _motion_lengths[motion_ids[e]]     */
  float dt;          /* _motion_dt[motion_ids[e]]          */
  int32_t num_frames;/* _motion_num_frames[motion_ids[e]]  */
  int32_t start_row; /* length_starts[motion_ids[e]]       */
} PhcEnvMotion;

PHC_API int phc_env_motion_gather(const PhcMotionLib* lib, const int64_t* motion_ids, int64_t n, PhcEnvMotion* out, void* stream);

/* Reset bookkeeping of the envs with mask != 0 in one launch (Humanoid._reset_envs / HumanoidIm._reset_task,
 * humanoid_im.py:955-1023): start_times = trunc(phase * len / (1/30)) * (1/30) (MotionLibBase.sample_time_interval,
 * motion_lib_base.py:414-423; phase = caller-supplied uniform [0,1) numbers), start_offsets / global_offset /
 * cycle_counter / progress / reset / terminate = 0.  cycle_counter, reset, terminate may be NULL. */
PHC_API int phc_reset_bookkeeping(const int64_t* mask, const float* phase, const PhcEnvMotion* env_motion, int64_t n,
                          float* start_times, float* start_offsets, float* global_offset /* [n,3] */, int32_t* cycle_counter,
                          int64_t* progress, int64_t* reset, int64_t* terminate, void* stream);

PHC_API int phc_motion_body_stride(int32_t num_bodies);        /* pass J + E for robots */
PHC_API int phc_motion_joint_stride(int32_t num_bodies);
PHC_API int phc_motion_dof_stride(int32_t num_dofs);           /* joint_stride of a hinge-joint robot: round_up(2*D, 4) */
/* Robot joint records: dof_pos[F, D], dof_vel[F, D] (motion_lib_real's dof_pos / dvs tables) -> frames_joint[F, dof_stride].
 * The body records of a robot are packed with phc_motion_pack(gts_t, grs_t, gvs_t, gavs_t, NULL, NULL, F, J + E, ...). */
PHC_API int phc_motion_pack_dofs(const float* dof_pos, const float* dof_vel, int64_t num_frames_total, int32_t num_dofs,
                         float* frames_joint, void* stream);

/* Pack the reference's separate tables into the records above (one pass, HBM-bound).
 * gts[F,J,3] grs[F,J,4] gvs[F,J,3] gavs[F,J,3] -> frames_body[F,body_stride];
 * lrs[F,J,4] dvs[F,J-1,3] -> frames_joint[F,joint_stride] (skipped when lrs/dvs/frames_joint is NULL). */
PHC_API int phc_motion_pack(const float* gts, const float* grs, const float* gvs, const float* gavs, const float* lrs,
                    const float* dvs, int64_t num_frames_total, int32_t num_bodies, float* frames_body,
                    float* frames_joint, void* stream);

/* Motion LOADER (SURVEY.md 8(f) rank 1): the per-clip CPU work of MotionLibSMPL.load_motion_with_skeleton
 * (phc/utils/motion_lib_smpl.py:101-180) for all clips of a (re)load in two launches -- heading randomisation (:141-149),
 * local rotations + forward kinematics (poselib/poselib/skeleton/skeleton3d.py:390-461), np.gradient / frame-to-frame
 * angle-axis velocities with scipy's gaussian_filter1d(sigma 2, "nearest") (skeleton3d.py:1100-1121) and
 * compute_motion_dof_vels (phc/utils/motion_lib_base.py:47-70).  Inputs are the on-disk clip arrays, concatenated over
 * clips, float64 as joblib yields them:
 *   pose_quat_global [F, J, 4] xyzw, root_trans [F, 3] ("root_trans_offset"), offsets [M, J, 3] = every clip's
 *   skeleton_tree.local_translation, parents [J] (-1 = root, parents[j] < j), heading [M] = angle about z in radians
 *   (the reference draws pi * (2 u - 1); NULL = flags.im_eval / flags.test: no randomisation), fps [M],
 *   length_starts / num_frames [M] (every clip needs >= 2 frames, as np.gradient does).
 * Outputs are the reference's float32 tables gts[F,J,3] grs[F,J,4] lrs[F,J,4] gvs[F,J,3] gavs[F,J,3] dvs[F,J-1,3]; feed them
 * to phc_motion_pack.  workspace: phc_motion_load_workspace_bytes(F, J) bytes, 16-byte aligned.  fix_trans_height (needs
 * the SMPL mesh model) is not part of this entry point: pass height-fixed translations. */
#define PHC_LOAD_MAX_BODIES 64
PHC_API int64_t phc_motion_load_workspace_bytes(int64_t num_frames_total, int32_t num_bodies);
PHC_API int phc_motion_load(const double* pose_quat_global, const double* root_trans, const double* offsets,
                    const int32_t* parents, const double* heading, const int64_t* length_starts, const int64_t* num_frames,
                    const double* fps, int64_t num_frames_total, int32_t num_motions, int32_t num_bodies, float* gts,
                    float* grs, float* lrs, float* gvs, float* gavs, float* dvs, void* workspace, void* stream);

/* MotionLibBase.get_motion_state (motion_lib_base.py:437-520, SMPL variant) for n arbitrary (id, time) queries:
 * frame bracket (_calc_frame_blend :549-559), lerp of pos/vel/angvel/dof_vel (+offset on pos), slerp of global
 * and local rotations, dof_pos = exp_map(local_rot[1:]).  Any output pointer may be NULL (skipped).
 * root_* are body 0 of rg_pos/rb_rot/body_vel/body_ang_vel. */
typedef struct PhcMotionStateOut {
  float* rg_pos;       /* [n, J, 3] */
  float* rb_rot;       /* [n, J, 4] */
  float* body_vel;     /* [n, J, 3] */
  float* body_ang_vel; /* [n, J, 3] */
  float* dof_pos;      /* [n, 3(J-1)] (SMPL) or [n, D] (robot) */
  float* dof_vel;      /* [n, 3(J-1)] (SMPL) or [n, D] (robot) */
  float* root_pos;     /* [n, 3] */
  float* root_rot;     /* [n, 4] */
  float* root_vel;     /* [n, 3] */
  float* root_ang_vel; /* [n, 3] */
  /* robots: the same four quantities for all J + E bodies (rg_pos_t, rg_rot_t, body_vel_t, body_ang_vel_t) */
  float* rg_pos_t;       /* [n, J+E, 3] */
  float* rg_rot_t;       /* [n, J+E, 4] */
  float* body_vel_t;     /* [n, J+E, 3] */
  float* body_ang_vel_t; /* [n, J+E, 3] */
} PhcMotionStateOut;

PHC_API int phc_motion_state(const PhcMotionLib* lib, const int64_t* motion_ids, const float* motion_times,
                     const float* offset /* [n,3] or NULL */, int64_t n, const PhcMotionStateOut* out, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Fused env step after physics: ONE kernel for
 *   Humanoid.post_physics_step (humanoid.py:1634-1650) ->
 *     HumanoidIm._compute_reward   (humanoid_im.py:873-948;  compute_imitation_reward :1523-1554, power :939-946)
 *     HumanoidIm._compute_reset    (humanoid_im.py:1117-1190; compute_humanoid_im_reset :1580-1608)
 *     HumanoidIm._compute_observations (humanoid_im.py:694-726): self obs compute_humanoid_observations_smpl_max
 *       (humanoid.py:1994-2050) + task obs compute_imitation_observations_v6 (humanoid_im.py:1308-1358)
 *     the two MotionLib queries those make (motion_lib_base.py:437-520) at t and t+dt
 *   HumanoidAMP.post_physics_step (humanoid_amp.py:194-210): _update_hist_amp_obs (:662-670) +
 *     build_amp_observations_smpl (:966-1011)
 * progress must already hold the incremented step counter (humanoid.py:1637).
 * ---------------------------------------------------------------------------------------------------------- */
#define PHC_MAX_EXT_BODIES 8
#define PHC_FLAG_UPRIGHT (1u << 0)         /* robot.has_upright_start                                   */
#define PHC_FLAG_LOCAL_ROOT_OBS (1u << 1)  /* env.local_root_obs                                        */
#define PHC_FLAG_ROOT_HEIGHT_OBS (1u << 2) /* env.root_height_obs (also the AMP root height column)     */
#define PHC_FLAG_POWER_REWARD (1u << 3)    /* env.power_reward -> reward_raw has 5 columns              */
#define PHC_FLAG_EARLY_TERM (1u << 4)      /* env.enableEarlyTermination                                */
#define PHC_FLAG_NO_COLLISION (1u << 5)    /* flags.no_collision_check                                  */
#define PHC_FLAG_TERM_USE_MEAN (1u << 6)   /* flags.im_eval and not strict_eval: mean-distance criterion */
#define PHC_FLAG_OBS_ONLY (1u << 7)        /* _compute_observations(env_ids) of the reset path: write obs (+ref_*) only */
#define PHC_FLAG_REWARD_FROM_CACHE (1u << 8) /* reward / reset read the reference pose from ref_cache (see PhcStepArgs) */
#define PHC_FLAG_SUBSET_REWARD (1u << 12)   /* env.full_body_reward: False -- tracking reward over the tracked bodies only */
#define PHC_FLAG_NO_SPECIALISE (1u << 11)  /* never take the compile-time specialised kernel (A/B runs, bit-identity tests) */
/* env_im_getup_mcp.yaml -- the configuration HumanoidImMCP trains in (time_steps 1, SMPL joints): */
#define PHC_FLAG_ZERO_OUT_FAR (1u << 9)   /* env.zero_out_far (zero_out_far_train False): point-goal reward mix (humanoid_im.py:890-905),
                                             task-obs overwrites for far references and the _point_goal update (:783-796) */
#define PHC_FLAG_CYCLE_MOTION (1u << 10)  /* env.cycle_motion: the launch runs _update_cycle_count (:1076-1079) and the clip
                                             wrap-around of _compute_reset (:1120-1146); pass_time = progress >= max_len - 1 */
/* env.obs_v: 7 -- the keypoint models (phc_kp_pnn_iccv, phc_kp_mcp_iccv, phc_comp_kp_2): */
#define PHC_FLAG_TASK_OBS_KP (1u << 13)  /* task obs compute_imitation_observations_v7 (humanoid_im.py:1362-1393, via _compute_task_obs
                                            :832-853) instead of v6: per sample [diff_pos 3K | diff_vel 3K | ref_pos - root 3K], heading-
                                            local, no rotations (9 K T columns).  zero_out_far overwrites positions of bodies 1.. and every
                                            velocity (:834-845); occlusion overwrites the position only -- the reference velocity stays
                                            (:847-851).  Built for <= PHC_LANE_BODIES bodies (PHC_ERR_UNSUPPORTED on the strided kernel). */
/* env.getup_schedule -- HumanoidImGetup / HumanoidImMCPGetup (phc/env/tasks/humanoid_im_getup.py), recovery episodes: */
#define PHC_FLAG_RECOVERY (1u << 14)     /* the launch runs _update_recovery_count of pre_physics_step (:198-201): recovery_counter =
                                            max(counter - 1, 0), written back; then, after the reset test (and the cycle_motion override),
                                            every env with counter > 0 gets reset = terminate = 0 -- also when the clip ran out (pass_time)
                                            -- and progress - 1 written back (:203-210).  Reward and reset see the incremented progress, the
                                            observation the decremented one (humanoid.py:1634-1647), so the ref_cache contract below holds.
                                            Step launches of time_steps 1, spherical-joint humanoids only (PHC_ERR_UNSUPPORTED otherwise);
                                            PHC_ERR_INVALID_ARG with PHC_FLAG_OBS_ONLY or a NULL recovery_counter. */
#define PHC_FLAG_AMP_CURRENT (1u << 15)  /* with PHC_FLAG_OBS_ONLY only: the observation-only launch also writes the AMP vector of the CURRENT
                                            simulator state (the row a step launch writes for the same state, bit for bit) into slot
                                            *ring_head (ring_head given) or slot 0 of amp_out: HumanoidAMP._compute_amp_observations(env_ids)
                                            (humanoid_amp.py:672-707) of the get-up reset path.  Same shapes as PHC_FLAG_RECOVERY. */

#define PHC_MAX_KEY_BODIES 8
#define PHC_MAX_BODIES 64      /* J + E; up to PHC_LANE_BODIES the staged one-body-per-lane kernels run, beyond it the strided
                                  ones (env_step_wide.cu: Unitree G1 38 + 1, SMPL-X 52) */
#define PHC_LANE_BODIES 32
#define PHC_MAX_AMP_JOINTS 64

typedef struct PhcStepArgs {
  /* ---- simulator state (inputs; contract of Humanoid._setup_tensors, humanoid.py:179-247) ---- */
  const float* body_state;  /* [N, bodies_per_env, 13]: pos rot vel ang_vel; only the first J bodies are read */
  const float* dof_state;   /* [N, D, 2] (pos, vel) interleaved, D = 3(J-1), or lib.num_dofs for robots          */
  const float* dof_force;   /* [N, D] or NULL when PHC_FLAG_POWER_REWARD is clear                              */
  int32_t bodies_per_env;
  /* ---- per-env motion bookkeeping ---- */
  const int64_t* progress;       /* [N] progress_buf                    */
  const int64_t* motion_ids;     /* [N] _sampled_motion_ids             */
  const PhcEnvMotion* env_motion;/* [N] optional pre-gathered parameters of motion_ids (phc_env_motion_gather); NULL = look up */
  /* read-only unless PHC_FLAG_CYCLE_MOTION is set: then a clip that wraps this step gets its re-based values written back */
  float* start_times;            /* [N] _motion_start_times             */
  float* start_offsets;          /* [N] _motion_start_times_offset      */
  float* global_offset;          /* [N,3] _global_offset                */
  int32_t* cycle_counter;        /* [N] _cycle_counter or NULL (is_recovery override, humanoid_im.py:1186-1188) */
  const int64_t* only_where;     /* [N] or NULL: when given, only envs with only_where[env] != 0 are processed (the
                                    reference's `env_ids` subset, kept as a mask so no host sync / nonzero() is needed) */
  PhcMotionLib lib;
  /* ---- configuration ---- */
  int32_t num_envs;   /* N */
  int32_t time_steps; /* T = _num_traj_samples (1 unless fut_tracks)  */
  float dt;           /* control dt (1/30)                            */
  float traj_dt;      /* _traj_sample_timestep (spacing of the T future samples) */
  uint32_t flags;     /* PHC_FLAG_*                                   */
  float k_pos, k_rot, k_vel, k_ang_vel; /* reward_specs (humanoid_im.py:57) */
  float w_pos, w_rot, w_vel, w_ang_vel;
  float power_coef;                     /* power_coefficient (humanoid_im.py:107) */
  float term_thresh[PHC_MAX_BODIES]; /* [J] termination distance per body, +inf for bodies outside reset_bodies (by
                                        value: configuration travels in the kernel parameters, not through a dependent load) */
  float term_dist_mean;      /* threshold of the first reset body (used by PHC_FLAG_TERM_USE_MEAN)       */
  /* robots: simulated pose of extend body e = body_rot[parent] * pos_in_parent + body_pos[parent], rotation = parent's
   * (humanoid_im.py:917-919); lib.num_ext_bodies entries */
  int32_t ext_parent[PHC_MAX_EXT_BODIES];
  float ext_pos[PHC_MAX_EXT_BODIES][3];
  int32_t num_key_bodies;
  int32_t key_bodies[PHC_MAX_KEY_BODIES]; /* _key_body_ids */
  int32_t amp_joints[PHC_MAX_AMP_JOINTS]; /* [num_amp_joints] joint indices (dof_subset / 3) kept in the AMP obs */
  int32_t num_amp_joints;
  /* ---- outputs ---- */
  float* obs;            /* [N, obs_stride] first 15J-3(+1) self obs then 24*J*T task obs (9*J*T with PHC_FLAG_TASK_OBS_KP) */
  int64_t obs_stride;    /* floats between rows                                                          */
  float* rew;            /* [N] rew_buf                                                                  */
  float* reward_raw;     /* [N, 5] (4 when power reward is off)                                          */
  int64_t* reset;        /* [N] reset_buf                                                                */
  int64_t* terminate;    /* [N] _terminate_buf                                                           */
  /* AMP observation.  amp_out[N, amp_out_stride]: the current step's vector (A floats) is written at slot 0.
   * If amp_hist_in != NULL the kernel also writes slots 1..S-1 = amp_hist_in slots 0..S-2 (newest-first window
   * shift of _update_hist_amp_obs); amp_hist_in may alias amp_out (in-place, like the reference) or be another
   * buffer (e.g. previous / current experience-buffer rows).  amp_out == NULL skips the AMP observation. */
  float* amp_out;
  const float* amp_hist_in;
  int64_t amp_out_stride; /* floats between env rows of amp_out and amp_hist_in (>= S*A)                 */
  int32_t amp_steps;      /* S                                                                            */
  /* optional side buffers of _compute_task_obs(save_buffer=True) (humanoid_im.py:855-868); NULL = skip */
  float* ref_body_pos;     /* [N, J, 3] */
  float* ref_body_rot;     /* [N, J, 4] */
  float* ref_body_vel;     /* [N, J, 3] */
  float* ref_body_ang_vel; /* [N, J, 3] */
  /* Interpolated reference pose kept across steps (SURVEY.md section 8d: "ref for reward time = 1248 B if the interpolated
   * pose from the previous step is kept").  [N, body_stride] rows of 13-float body records (pos3 rot4 vel3 angvel3, global
   * offset included), 16-byte aligned.  When non-NULL every launch writes the pose it interpolated for the FIRST observation
   * sample, i.e. for motion time (progress+1)*dt + start + offset.  With PHC_FLAG_REWARD_FROM_CACHE the launch takes the
   * reference pose of the reward / reset test from here instead of interpolating the bracket of progress*dt + start +
   * offset: valid exactly when the previous launch (step or PHC_FLAG_OBS_ONLY reset launch) of that env ran with
   * progress-1 and the same start / offset / clip -- which HumanoidIm's step / reset sequence guarantees.  The values
   * are bit-identical to re-interpolating.  ref_body_* above are then strided views of it (columns 0:3, 3:7, 7:10, 10:13). */
  float* ref_cache;
  /* ---- PHC_FLAG_ZERO_OUT_FAR / PHC_FLAG_CYCLE_MOTION (appended; ignored when both flags are clear) ---- */
  float close_distance;        /* env.close_distance (0.25): beyond it the task obs sees the simulated pose as reference   */
  float far_distance;          /* env.far_distance (3): beyond it the reference root becomes a direction of this length    */
  int32_t max_episode_length;  /* env.episode_length                                                                       */
  float* point_goal;           /* [N] _point_goal: read by the reward (previous distance), rewritten by the observation    */
  const float* cycle_phase;    /* [N] uniform [0,1) numbers: sample_time_interval's draw for a clip that wraps this step   */
  /* ---- flags.im_eval extras of HumanoidIm.post_physics_step (humanoid_im.py:674-680); NULL = skip ---- */
  float* mpjpe;                /* [N] mean over the J bodies of |body_pos - reference pos| at the current motion time      */
  float* body_pos_gt;          /* [N, J, 3] that reference pose's positions (extras['body_pos_gt'])                        */
  /* ---- AMP ring with the head kept ON THE DEVICE (appended; NULL = the host passes amp_out already offset to the slot) ----
   * When non-NULL, amp_out is the ring base and this step's vector goes to slot *ring_head of every env.  Lets a whole rollout
   * (whose slot changes every step) be captured once as a CUDA graph; phc_ring_advance moves the head between steps. */
  const int32_t* ring_head;
  /* ---- tracked-body subsets, occlusion training, shape columns (appended; all zero / NULL = the plain full-body configuration) ----
   * env.trackBodies (humanoid_im.py:64-66, :762-770; env_vr.yaml:38-39: Head + both hands): the task observation is built over the
   * K = num_track tracked bodies only (24 K T columns, body j sits at position track_slot[j]); with PHC_FLAG_SUBSET_REWARD
   * (env.full_body_reward: False, :926-935) the tracking reward averages over the same subset.  occlusion [N, K] (uint8; K = J when
   * num_track == 0) is random_occlu_idx of _occl_training (:797-804): an occluded tracked body shows the SIMULATED pose as its
   * reference in the task observation.  shape_params [N, num_shape] / limb_weights [N, num_limb] are the has_shape_obs /
   * has_limb_weight_obs columns appended to the self observation (humanoid.py:2043-2047; robot/smpl_humanoid_shape.yaml). */
  int32_t num_track;
  int8_t track_slot[PHC_MAX_BODIES];
  const uint8_t* occlusion;
  const float* shape_params;
  int32_t num_shape;
  const float* limb_weights;
  int32_t num_limb;
  /* ---- PHC_FLAG_RECOVERY (appended; ignored when the flag is clear) ----
   * _recovery_counter [N] of HumanoidImGetup (humanoid_im_getup.py:61), read and rewritten by the launch.  With the flag set the
   * launch also WRITES progress (declared const above for every other launch): progress - 1 for the envs still recovering. */
  int32_t* recovery_counter;
} PhcStepArgs;

/* Sizes implied by a configuration (so callers can allocate): */
PHC_API int phc_self_obs_dim(int32_t num_bodies, uint32_t flags);                    /* 1 + 15J - 3          */
PHC_API int phc_task_obs_dim(int32_t num_bodies, int32_t time_steps);                /* 24 J T               */
PHC_API int phc_task_obs_dim_flags(int32_t num_bodies, int32_t time_steps, uint32_t flags); /* 9 J T with PHC_FLAG_TASK_OBS_KP, else 24 J T */
PHC_API int phc_amp_obs_dim(int32_t num_amp_joints, int32_t num_key_bodies, uint32_t flags); /* 13 + 9 nj + 3 nk */
/* build_amp_observations_robot (humanoid_amp.py:1062-1104): [root_h?, rot6, vel3, ang_vel3, dof_pos[D], dof_vel[D], key 3 nk] */
PHC_API int phc_amp_obs_dim_robot(int32_t num_dofs, int32_t num_key_bodies, uint32_t flags); /* 13 + 2 D + 3 nk */

PHC_API int phc_env_step(const PhcStepArgs* args, void* stream);
/* How many phc_env_step calls of this process took the compile-time specialised kernel of the shipped SMPL steady state
 * (flags = UPRIGHT | LOCAL_ROOT_OBS | ROOT_HEIGHT_OBS | POWER_REWARD | EARLY_TERM | REWARD_FROM_CACHE, env_motion and ref_cache
 * given, no env mask, no ref_body_* buffers, AMP ring slot / obs rows / pose cache movable as 16-byte granular bulk copies).
 * Diagnostic: lets a caller (and the tests) see that its buffers qualify.  PHC_ENV_FAST=0 in the environment disables it. */
PHC_API int64_t phc_env_step_fast_launches(void);
/* phc_env_step is launched with programmatic stream serialisation (PDL): its CTAs may become resident, and set up their shared
 * memory barriers, while the previous kernel of the stream is finishing; the kernel executes griddepcontrol.wait before its first
 * global-memory access, so ordering is exactly that of a plain launch.  PHC_ENV_PDL=0 in the environment switches the attribute off. */

/* ------------------------------------------------------------------------------------------------------------
 * Get-up schedule (HumanoidImGetup, phc/env/tasks/humanoid_im_getup.py): reset selection of the envs with mask != 0, in ONE
 * launch and without a host sync (CUDA-graph capturable), in the order of _reset_actors (:135-182):
 *   1. available[assignment[e]] = 0 for every masked env (assignments are never cleared: a stale one frees a state another env
 *      may hold, as in the reference);
 *   2. recovery envs: u_rec[e] < *p_rec and terminate[e] == 1 -> counter = recovery_steps, simulator state untouched;
 *   3. fall envs, among the rest: u_fall[e] < *p_fall.  The k-th fall env in ascending env order takes the k-th state s with
 *      available[s] == 0 in the order of perm (a permutation of [0, P)): body_state[e, 0] = fall_root[s] (13 floats),
 *      dof_state[e] = (fall_dof_pos[s], 0), counter = recovery_steps, available[s] = 1, assignment[e] = s;
 *   4. everything else: ref_init[e] = 1 (feed it to phc_reset_bookkeeping / phc_set_env_state / phc_amp_obs_demo) and counter = 0;
 *   5. progress / reset / terminate = 0 for fall and recovery envs (phc_reset_bookkeeping clears the ref-init ones).
 * ref_init / fall (int64 0/1) are written for every env (0 outside the mask).  torch.bernoulli(p) == 1 is u < p; perm drawn uniformly
 * gives the law of available_ids[randperm(n)].  p_rec / p_fall live in device memory so that a captured launch sees schedule
 * changes.  The bank size P must equal N (then a fall env always finds a free state).  D = dofs per env. */
PHC_API int phc_getup_reset(const int64_t* mask, const int64_t* terminate_in, const float* u_rec, const float* u_fall, const int64_t* perm,
                    const float* p_rec, const float* p_fall, int32_t recovery_steps, const float* fall_root /* [P,13] */,
                    const float* fall_dof_pos /* [P,D] */, int64_t num_states, int64_t* available, int64_t* assignment,
                    int32_t* recovery_counter, int64_t n, float* body_state, int32_t bodies_per_env, float* dof_state, int32_t num_dofs,
                    int64_t* progress, int64_t* reset, int64_t* terminate, int64_t* ref_init, int64_t* fall, void* stream);
/* _init_amp_obs_default (humanoid_amp.py:570-573) on the AMP ring: for every env with mask != 0, every slot of its ring row =
 * slot *head (the newest vector, e.g. what a PHC_FLAG_AMP_CURRENT launch wrote). */
PHC_API int phc_amp_ring_fill(float* ring, int64_t ring_stride, int64_t n, int32_t num_steps, int32_t amp_dim, const int32_t* head_dev,
                      const int64_t* mask, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Imitation evaluation metrics: the per-step part of IMAmpAgent._post_step_eval (phc/learning/im_amp.py:244-363) and of smpl_sim's
 * compute_metrics_lite, which the reference runs on the host over the per-clip slices [:num_steps - 1] of the stacked
 * body_pos / body_pos_gt.  ONE launch per eval step, no host sync.  For env e, with d_t = body_pos[e] - body_pos_gt[e] ([J, 3]):
 *   frame t counts when t < num_steps[e] - 1 (the slice); then, with means over the J bodies,
 *   acc[e, 0] += mean |d_t[j]|                               mpjpe_g
 *   acc[e, 1] += mean |d_t[j] - d_t[0]|                      mpjpe_l (root-relative)
 *   acc[e, 2] += mean |a R^T y_j + mu_gt - gt_j|             mpjpe_pa: pred aligned onto gt by the similarity transform with a
 *                                                            proper rotation (VideoPose3D's p_mpjpe: SVD, det(R) = -1 sign fix)
 *   acc[e, 3] += mean |d_t[j] - d_{t-1}[j]|        (t >= 1)  vel_dist   = |(p_t - p_{t-1}) - (g_t - g_{t-1})|
 *   acc[e, 4] += mean |d_t - 2 d_{t-1} + d_{t-2}|  (t >= 2)  accel_dist
 *   acc[e, 5..7] += 1 for the frames counted in 0-2, 3 and 4.
 * Sums are in the units of the positions (metres; compute_metrics_lite reports millimetres), fp64, added in a fixed order (no
 * atomics): bit-identical from run to run.  d_t is written to ring[t & 1] on every step; ring[(t + 1) & 1] must hold d_{t-1} for
 * t >= 1 and ring[t & 1] d_{t-2} for t >= 2, i.e. call once per step with t = 0, 1, 2, ... (t restarts at 0 for a new batch of
 * clips, the ring needs no reset).  body_pos: element (e, j, c) at e * env_stride + j * body_stride + c * coord_stride floats
 * (coord_stride must be 1; e.g. the [..., :J, 0:3] view of the [N, B, 13] rigid-body state); body_pos_gt [n, J, 3] contiguous;
 * num_steps [n] int32 (get_motion_num_steps()); ring [2, n, J, 3] fp32; acc [n, PHC_EVAL_ACC_FIELDS] fp64.  1 <= J <= 64, n >= 1. */
#define PHC_EVAL_ACC_FIELDS 8
PHC_API int phc_eval_metrics_step(const float* body_pos, int64_t env_stride, int64_t body_stride, int64_t coord_stride,
                                  const float* body_pos_gt, const int32_t* num_steps, int32_t t, int64_t n, int32_t num_bodies,
                                  float* ring, double* acc, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Episode statistics of the rollout: the per-step bookkeeping of AMPAgent.play_steps (phc/learning/amp_agent.py:358-369) with
 * rl_games 1.1.4's AverageMeter, ONE launch per step, no host sync.  For every env i (dones: the int64 reset flags):
 *   v_r = cur_r[i] + rewards[i], v_l = cur_l[i] + 1; cur_r[i] = v_r * (1 - done), cur_l[i] = v_l * (1 - done)   (fp32)
 * and, when k = #(done != 0) > 0, the meters m = 0 (game_rewards, values v_r) and m = 1 (game_lengths, values v_l) of the done envs:
 *   new_mean = mean of the k values; size = min(k, games_to_track); old = min(games_to_track - size, meter_size[m])
 *   meter_mean[m] = (meter_mean[m] * old + new_mean * size) / (old + size); meter_size[m] = old + size
 * rewards, cur_r, cur_l [n] fp32; dones [n] int64; meter_mean [2] fp32; meter_size [2] int32.  Fixed-order sums (fp64), no
 * atomics: bit-identical from run to run.  n >= 1, games_to_track >= 1. */
PHC_API int phc_episode_stats(const float* rewards, const int64_t* dones, int64_t n, float* cur_r, float* cur_l, float* meter_mean,
                              int32_t* meter_size, int32_t games_to_track, void* stream);

/* build_amp_obs_demo (humanoid_amp.py:253-284) and the history re-initialisation of _init_amp_obs_ref
 * (:575-603): AMP observations of the REFERENCE motion at t0 - (first_step + k)*dt, k = 0..num_steps-1,
 * written to out[n, num_steps, A] (row stride out_stride floats).  Needs lib->frames_joint. */
PHC_API int phc_amp_obs_demo(const PhcMotionLib* lib, const int64_t* motion_ids, const float* times0, int64_t n,
                     int32_t first_step, int32_t num_steps, float dt, uint32_t flags, const int32_t* key_bodies /* host */,
                     int32_t num_key_bodies, const int32_t* amp_joints /* host */, int32_t num_amp_joints, float* out,
                     int64_t out_stride, const int64_t* only_where /* [n] or NULL: skip rows whose entry is 0 */,
                     int32_t slot_offset /* ring rotation: step k lands in slot (k + slot_offset) % num_steps; 0 = plain */,
                     void* stream);

/* AMP observation ring.  Instead of shifting the [S, A] window of every env each step (2 x 7 KB per env-step,
 * humanoid_amp.py:662-670) the fused step writes only the newest vector into physical slot `head` of a ring
 * (phc_env_step with amp_out = ring + head*A, amp_hist_in = NULL), and the newest-first window the agent stores
 * (extras['amp_obs'], amp_agent.py:341) is produced by this copy straight into its destination:
 *   out[n, k, :] = ring[n, (head + k) % S, :]. */
PHC_API int phc_amp_window_export(const float* ring, int64_t ring_stride, int64_t n, int32_t num_steps, int32_t amp_dim,
                          int32_t head, float* out, int64_t out_stride, void* stream);

/* The same two calls with the ring rotation / head read from DEVICE memory (`*_dev` non-NULL overrides the integer argument),
 * and the one-thread kernel that moves the head one slot back before a step: *head = (*head - 1 + num_slots) % num_slots. */
PHC_API int phc_amp_obs_demo_ring(const PhcMotionLib* lib, const int64_t* motion_ids, const float* times0, int64_t n,
                          int32_t first_step, int32_t num_steps, float dt, uint32_t flags, const int32_t* key_bodies,
                          int32_t num_key_bodies, const int32_t* amp_joints, int32_t num_amp_joints, float* out, int64_t out_stride,
                          const int64_t* only_where, int32_t slot_offset, const int32_t* slot_offset_dev, void* stream);
PHC_API int phc_amp_window_export_ring(const float* ring, int64_t ring_stride, int64_t n, int32_t num_steps, int32_t amp_dim,
                               int32_t head, const int32_t* head_dev, float* out, int64_t out_stride, void* stream);
PHC_API int phc_ring_advance(int32_t* head, int32_t num_slots, void* stream);
/* adds n to the launch counter phc_launch_count() reports (a replayed CUDA graph launches kernels the library did not see) */
PHC_API void phc_launch_count_add(int64_t n);

/* Reset path (HumanoidAMP._set_env_state, humanoid_amp.py:605-637 fed by _sample_ref_state, humanoid_im.py:1000-1023):
 * write the reference pose at (motion_ids[e], times[e]) (+offset) into the simulator tensors of every env e with
 * only_where[e] != 0 (NULL = all): body_state[e, 0:J, 13] and, when dof_state != NULL, dof_state[e, :, (pos, vel)]. */
PHC_API int phc_set_env_state(const PhcMotionLib* lib, const int64_t* motion_ids, const float* times, const float* offset,
                      const int64_t* only_where, int64_t n, float* body_state, int32_t bodies_per_env, float* dof_state,
                      void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * PPO scalars
 * ---------------------------------------------------------------------------------------------------------- */
/* CommonAgent.discount_values (phc/learning/common_agent.py:493-505) + returns = advs + values
 * (amp_agent.py:384-385).  Time-major [T, N] fp32 inputs (the reference's [T,N,1] tensors are the same memory);
 * advs / returns may be NULL individually. */
PHC_API int phc_gae(const float* fdones, const float* values, const float* rewards, const float* next_values, int32_t horizon,
            int64_t num_envs, float gamma, float tau, float* advs, float* returns, void* stream);

/* CommonAgent._calc_advs (common_agent.py:589-599): adv = returns - values, then (adv-mean)/(std+1e-8) with the
 * UNBIASED std over all n elements.  workspace: >= phc_adv_norm_workspace_bytes(n) bytes of device scratch. */
PHC_API int64_t phc_adv_norm_workspace_bytes(int64_t n);
PHC_API int phc_adv_norm(const float* returns, const float* values, int64_t n, int32_t normalize, float* advs,
                 void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * MLP building blocks (actor / critic / discriminator are nn.Linear stacks: phc/learning/network_builder.py:105-124,
 * amp_network_builder.py:58-249; fp32 in the reference -> computed fp32-equivalent on the tensor cores, 3xTF32)
 * ---------------------------------------------------------------------------------------------------------- */
/* Activation codes of the GEMM epilogues (`act` argument; nn.ReLU of im.yaml, nn.SiLU of im_big.yaml / im_pnn_big.yaml /
 * im_mcp_big.yaml).  `aux` [M, ldaux] is optional:
 *   PHC_ACT_NONE / PHC_ACT_RELU with aux : ReLU backward, out *= (aux > 0)        (aux = the layer's output, read)
 *   PHC_ACT_SILU                         : out = x * sigmoid(x); aux (if given) receives the pre-activation x (written)
 *   PHC_ACT_SILU_BWD (aux required)      : out *= d silu / dx at x = aux          (aux = the saved pre-activation, read) */
#define PHC_ACT_NONE 0
#define PHC_ACT_RELU 1
#define PHC_ACT_SILU 2
#define PHC_ACT_SILU_BWD 3
/* phc_gemm_tc5s / phc_gemm_group only -- the ReLU mask as ONE BIT per element instead of re-reading the fp32 activations in
 * the backward pass (32x less traffic): aux is then a uint32 array [M, ldaux] (ldaux in words, >= ceil(N / 32)), bit j of
 * word (m, n / 32) belongs to column n = 32 * (n / 32) + j.
 *   PHC_ACT_RELU_BITS : out = relu(x); aux (optional) receives the bits (x > 0)
 *   PHC_ACT_MASK_BITS : out *= bit     (aux required, read) */
#define PHC_ACT_RELU_BITS 4
#define PHC_ACT_MASK_BITS 5
/* C[M,N] (+)= epi(alpha * sum_k A(m,k) B(n,k)).  a_kmajor: A(m,k) = A[m*lda + k] (else A[k*lda + m]); b_kmajor: B(n,k) =
 * B[n*ldb + k] (else B[k*ldb + n]).  Forward Y = X W^T: (1,1); input gradient dX = dY W: (1,0); weight gradient
 * dW = dY^T X: (0,0).  Epilogue in order: *alpha, +bias[n], activation `act` / aux (above), then store or atomic
 * accumulate (accumulate != 0; required for k_splits > 1, C pre-zeroed, linear epilogue only).
 * A, B 16-byte aligned, lda/ldb multiples of 4 and >= the contiguous extent rounded up to 4 (zero padded). */
PHC_API int phc_gemm(const float* A, int64_t lda, int32_t a_kmajor, const float* B, int64_t ldb, int32_t b_kmajor, float* C,
             int64_t ldc, int32_t M, int32_t N, int32_t K, float alpha, const float* bias, int32_t act,
             float* aux, int64_t ldaux, int32_t accumulate, int32_t k_splits, void* stream);
/* Hopper tensor-core variant of phc_gemm (wgmma kind tf32, gemm_wgmma.cu).  Same epilogue contract.  3xTF32 with each
 * operand pre-split once by phc_split_tf32 (hi = rna_tf32(x), lo = rna_tf32(x - hi)); hi and lo share the leading
 * dimension.  All four operand arrays 16-byte aligned, lda/ldb multiples of 4; C 8-byte aligned, ldc even. */
PHC_API int phc_split_tf32(const float* x, int64_t ldx, int64_t rows, int32_t cols, float* hi, float* lo, int64_t ldo, void* stream);
PHC_API int phc_gemm_tc5(const float* A_hi, const float* A_lo, int64_t lda, int32_t a_kmajor, const float* B_hi, const float* B_lo,
                 int64_t ldb, int32_t b_kmajor, float* C, float* C_hi /* optional: split copies of C for the next GEMM */,
                 float* C_lo, int64_t ldc, int32_t M, int32_t N, int32_t K, float alpha, const float* bias, int32_t act,
                 float* aux, int64_t ldaux, int32_t accumulate, int32_t k_splits, void* stream);
/* The same GEMM with the 3xTF32 operand split done in SHARED memory (gemm_wgmma.cu): plain fp32 operands, no pre-split
 * copies.  A, B, C 16-byte aligned; lda, ldb, ldc multiples of 4.
 * phc_gemm_group runs up to PHC_GEMM_GROUP_MAX independent problems (e.g. the same layer of actor, critic and
 * discriminator: network_builder.py:105-124 builds three separate nn.Sequential stacks that the reference evaluates one
 * after the other) as ONE persistent launch over the union of their tiles.
 * Reproducibility: split-K slices add into C in slice order, and problems of one launch that accumulate into the SAME C (same
 * pointer, M, N and ldc) add one after the other in problem order, each with its slices in order; the result is the same bit for
 * bit from run to run.  Write hazards are refused (PHC_ERR_INVALID_ARG): the spans [C, C + (M-1)*ldc + N) of two non-empty
 * problems of one launch must not overlap, except for such a same-C accumulating group. */
#define PHC_GEMM_GROUP_MAX 8
typedef struct PhcGemmDesc {
  const float* A; int64_t lda; int32_t a_kmajor;
  const float* B; int64_t ldb; int32_t b_kmajor;
  float* C; int64_t ldc;
  int32_t M, N, K;
  float alpha;
  const float* bias;        /* optional [N] */
  int32_t act;              /* PHC_ACT_* */
  float* aux; int64_t ldaux;
  int32_t accumulate, k_splits;
  const float* B_lo;        /* optional: the 3xTF32 low part of B, same layout and ldb, made by phc_split_lo; validated and not
                             * read (the kernel makes the identical low part from the tiles it stages) */
  const float* B_img;       /* optional: B's weight image for this problem's N and K (phc_gemm_make_images), 16-byte aligned, with
                             * a_kmajor or A_img.  With 128 x 128 tiles the kernel then reads B from the image (one bulk copy per
                             * k-block) and A straight into the tensor-core registers instead of staging both; the result is the
                             * same bit for bit.  128 x 256 tiles and PHC_GEMM_TF32_SINGLE_PASS ignore it.  The image must be
                             * remade whenever B changes. */
  const float* A_img;       /* optional, only with B_img: A's image in the same layout with rows = M (phc_gemm_make_images with
                             * B = A, N = M, b_kmajor = a_kmajor), 16-byte aligned.  With both images the kernel reads both operands
                             * by bulk copy and never looks at a_kmajor / b_kmajor; the result is again the same bit for bit, and
                             * the same two cases ignore both images.  Meant for the weight gradient (dW += dY^T X, both operands
                             * mn-major activations), whose images are made once per launch instead of staged once per tile. */
  float* C_img;             /* optional: the epilogue also writes the image of the stored output with rows = M and K = N (the
                             * layout phc_gemm_make_images makes from C with b_kmajor = 1, bit for bit, zero outside M x N), so that
                             * the next layer's forward or input-gradient GEMM can take C as its A_img without a separate pass.
                             * 16-byte aligned, phc_gemm_image_floats(M, N) floats.  Refused with accumulate, k_splits > 1, 128 x 256
                             * tiles and PHC_GEMM_TF32_SINGLE_PASS. */
} PhcGemmDesc;
/* Weight image of a B operand (B(n,k) as in PhcGemmDesc, N x K): one block of 8192 floats per (128-row n-tile nt, 32-wide k-block
 * kb), block nt * ceil(K / 32) + kb, each block [hi | lo] of 4096 floats with hi = trunc_tf32(B), lo = rna_tf32(B - hi) (the
 * split the GEMM makes itself); inside a half, element (n, k) of the tile sits at float 256 (n / 8) + 32 (k / 4) + 4 (n % 8) + k % 4
 * (8-row x 16-byte core matrices, K-major, no swizzle).  Zero outside N x K.  phc_gemm_image_floats(N, K) is its size.
 * phc_gemm_make_images writes `count` images in one launch (more than 64 take one launch per 64). */
typedef struct PhcGemmImageDesc {
  const float* B; int64_t ldb; int32_t b_kmajor;
  int32_t N, K;
  float* img;
} PhcGemmImageDesc;
PHC_API int64_t phc_gemm_image_floats(int32_t N, int32_t K);
PHC_API int phc_gemm_make_images(const PhcGemmImageDesc* images, int32_t count, void* stream);
/* lo[i] = rna_tf32(x[i] - trunc_tf32(x[i])): the second TF32 term of every fp32 value, what the GEMM computes per staged tile */
PHC_API int phc_split_lo(const float* x, float* lo, int64_t n, void* stream);
PHC_API int phc_gemm_group(const PhcGemmDesc* problems, int32_t count, void* stream);
PHC_API int phc_gemm_tc5s(const float* A, int64_t lda, int32_t a_kmajor, const float* B, int64_t ldb, int32_t b_kmajor, float* C,
                  int64_t ldc, int32_t M, int32_t N, int32_t K, float alpha, const float* bias, int32_t act,
                  float* aux, int64_t ldaux, int32_t accumulate, int32_t k_splits, void* stream);
/* Arithmetic of phc_gemm_tc5s / phc_gemm_group (process-wide switch, read at launch):
 *   PHC_GEMM_FP32_3XTF32      (default) three tensor-core products per fp32 product, fp32-equivalent (the parity path: the
 *                             reference trains with mixed_precision: False);
 *   PHC_GEMM_TF32_SINGLE_PASS one tensor-core tf32 product: operands truncated to 10 mantissa bits, fp32 accumulate, ~1e-3
 *                             relative -- the reduced-precision tensor-core mode BASELINE.json configs[3] asks for (bf16-class: the
 *                             same 8-bit exponent, 3 more mantissa bits than bf16), 3x fewer tensor instructions and no split pass.
 *                             OPT-IN, with its own tolerance (tests/test_gpu_gemm_tc5s.py); nothing in the parity tests uses it. */
#define PHC_GEMM_FP32_3XTF32 0
#define PHC_GEMM_TF32_SINGLE_PASS 1
PHC_API int phc_gemm_set_precision(int32_t mode);
/* CTAs per tile (tests / tools): 0, 1 or 2 are accepted; every tile is computed by one CTA */
PHC_API int phc_gemm_tc5s_set_ctas(int32_t ctas);
/* tile shape (tests / tools): 128 = 128 x 128 x 32 tiles (default), 256 = 128 x 256 x 16 tiles, 0 = back to the default */
PHC_API int phc_gemm_tc5s_set_tile(int32_t width);
/* tile order (tests / tools): 1 = tiles drawn from a global counter (default; env PHC_TC5S_SCHED=static turns it
 * off), 0 = static striding (tile t on CTA t mod grid), -1 = back to the default */
PHC_API int phc_gemm_tc5s_set_sched(int32_t mode);
/* Humanoid._action_to_pd_targets (phc/env/tasks/humanoid.py:1711-1713) as pre_physics_step applies it (:1540-1556):
 *   out[e, d] = pd_action_offset[d] + pd_action_scale[d] * action(e, d)        (product rounded, then the sum)
 * dof_of_action (device int32 [num_dofs], optional): reduce_action -- the action column that drives dof d, or -1 (action 0);
 * NULL needs num_actions == num_dofs.  zero_mask (device uint8 [num_dofs], optional): dofs forced to 0 afterwards
 * (_freeze_hand / _freeze_toe).  The result is what the backend hands to gym.set_dof_position_target_tensor. */
PHC_API int phc_pd_targets(const float* actions, int64_t lda, int64_t n, int32_t num_dofs, int32_t num_actions,
                   const int32_t* dof_of_action, const float* offset, const float* scale, const uint8_t* zero_mask,
                   float* out, int64_t ldo, void* stream);
/* out[n] (+)= alpha * sum_m X[m*ld + n]   (bias gradients) */
PHC_API int phc_colsum(const float* X, int64_t ld, int32_t M, int32_t N, float alpha, float* out, int32_t accumulate,
               void* stream);
/* the same for up to PHC_GEMM_GROUP_MAX matrices in ONE launch (the bias gradients of all stacks at one layer depth):
 * out[n] += alpha * sum_m X[m, n] (always accumulating: `out` holds zeros or earlier contributions).  X 16-byte aligned, ld a multiple
 * of 4 floats and >= N rounded up to 4 (the 4-padded activation workspaces). */
/* out[n] += alpha * sum_m X[m, n] for each problem, the row blocks added in a fixed order; the problems' out ranges must not overlap */
typedef struct PhcColsumDesc { const float* X; int64_t ld; int32_t M, N; float alpha; float* out; } PhcColsumDesc;
PHC_API int phc_colsum_group(const PhcColsumDesc* problems, int32_t count, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Learner-side element-wise / reduction kernels (between the GEMMs of the PPO + AMP update)
 * ---------------------------------------------------------------------------------------------------------- */
/* RunningMeanStd.forward (phc/utils/running_mean_std.py:69-109): y = clamp((x-mean)/sqrt(var+eps), -5, 5), or with
 * unnorm != 0: y = sqrt(var+eps)*clamp(x,-5,5)+mean.  fp64 stats, fp32 data; only columns [0,d) are written. */
PHC_API int phc_rms_apply(const float* x, int64_t ldx, int64_t n, int32_t d, const double* mean, const double* var, float eps,
                  int32_t unnorm, float* y, int64_t ldy, const int64_t* row_idx /* [n] or NULL: y[r] = f(x[row_idx[r]]),
                  the minibatch gather of AMPDataset._get_item (amp_datasets.py:81-94) fused in */, void* stream);
/* ... and its train-mode statistics update (parallel-variance merge of the batch mean / unbiased var, :56-68). */
/* phc_rms_apply (with mean_apply / var_apply: the live statistics, or the frozen copy of AMPAgent._preproc_obs(use_temp), amp_agent.py:535-552)
 * and phc_rms_update of the live statistics (mean, var, count) in ONE pass over the gathered rows: RunningMeanStd.forward in train mode
 * normalises with the statistics as they are and folds the batch in afterwards (running_mean_std.py:99-107).  mean_apply may alias mean. */
PHC_API int phc_rms_apply_update(const float* x, int64_t ldx, int64_t n, int32_t d, const double* mean_apply, const double* var_apply, float eps,
                         float* y, int64_t ldy, const int64_t* row_idx, double* mean, double* var, double* count, void* workspace,
                         void* stream);
/* device scratch of phc_rms_update / phc_rms_apply_update: one fp64 (sum, sum of squares) pair per column and row strip, the strips
 * added in a fixed order, so the statistics do not depend on scheduling */
PHC_API int64_t phc_rms_workspace_bytes(int32_t d);
PHC_API int phc_rms_update(const float* x, int64_t ldx, int64_t n, int32_t d, double* mean, double* var, double* count,
                   void* workspace, const int64_t* row_idx /* [n] or NULL, as in phc_rms_apply */, void* stream);
/* rl_games ModelA2CContinuousLogStd (is_train False): action = mu + exp(logstd)*noise, neglogp of that action;
 * mus / sigmas (optional) are the copies the experience buffer stores. */
PHC_API int phc_gaussian_sample(const float* mu, int64_t ldmu, const float* logstd, const float* noise, int64_t n, int32_t A,
                        float* actions, float* neglogp, float* mus, float* sigmas, void* stream);
/* Actor side of AMPAgent.calc_gradients (amp_agent.py:604-641): neglogp of the stored actions, CommonAgent._actor_loss
 * (common_agent.py:564-574), bound_loss (:512-520), policy_kl; writes d(total loss)/d(mu) = inv_batch * (...).
 * stats (float[16], caller-zeroed, sums over rows): [0] actor loss [1] bound loss [2] clipped count [3] kl [4] entropy
 * Every `stats` / `stat` sum of the kernels below is added in a fixed order (per-block partials, then the blocks in order), so it
 * is the same bit for bit from run to run; launches that add into the same statistic must be ordered (one stream). */
PHC_API int phc_ppo_actor_grad(const float* mu, int64_t ldmu, const float* logstd, const float* actions,
                       const float* old_neglogp, const float* adv, const float* old_mu, const float* old_sigma, int64_t n,
                       int32_t A, float e_clip, float bound_coef, float inv_batch, float* dmu, int64_t lddmu, float* stats,
                       void* stream);
/* CommonAgent._critic_loss with clip_value False (:576-587): dv = coef*2*(v-ret)*inv_batch; stats[5] += sum (ret-v)^2 */
PHC_API int phc_ppo_critic_grad(const float* v, int64_t ldv, const float* ret, int64_t n, float coef, float inv_batch, float* dv,
                        int64_t lddv, float* stats, void* stream);
/* phc_ppo_actor_grad + phc_ppo_critic_grad on an INDEX-COMPOSED minibatch: actions / old_neglogp / adv / old_mu / old_sigma / ret are the
 * epoch's dataset arrays ([batch_size, ...], AMPDataset.values_dict, amp_datasets.py:81-101) and minibatch row r is their row row_idx[r];
 * mu / v / dmu / dv are in minibatch order.  Replaces six gather passes (`values_dict[k][idx]`) per minibatch. */
PHC_API int phc_ppo_grads_gather(const float* mu, int64_t ldmu, const float* logstd, const float* actions, const float* old_neglogp,
                         const float* adv, const float* old_mu, const float* old_sigma, const float* v, int64_t ldv, const float* ret,
                         const int64_t* row_idx, int64_t n, int32_t A, float e_clip, float bound_coef, float critic_coef, float inv_batch,
                         float* dmu, int64_t lddmu, float* dv, int64_t lddv, float* stats, void* stream);
/* AMPAgent._disc_loss prediction part (amp_agent.py:739-743, :791-804): rows [0,n_agent) are agent+replay logits
 * (target 0), rows [n_agent, n_agent+n_demo) demo logits (target 1); dlogit = coef*0.5*dBCE/n.
 * stats[6] += sum softplus(agent) [7] += sum softplus(-demo) [8] += #(agent<0) [9] += #(demo>0)
 * [13] += sum agent logit [14] += sum demo logit (stats must hold at least 15 floats) */
PHC_API int phc_disc_logit_grad(const float* logit, int64_t ld, int64_t n_agent, int64_t n_demo, float coef, float* dlogit,
                        int64_t ldd, float* stats, void* stream);
/* AMPAgent._calc_disc_rewards (:864-878) (+ _combine_rewards :848-853 when combined != NULL) */
PHC_API int phc_disc_reward(const float* logit, int64_t ld, const float* task_rewards, int64_t n, float scale, float w_task,
                    float w_disc, float* disc_rewards, float* combined, void* stream);
/* u[b,j] = h[b,j] > 0 ? w[j] : 0 : first factor of d(logit)/d(input) through a ReLU MLP (gradient penalty, :749-768) */
PHC_API int phc_relu_mask_row(const float* h, int64_t ldh, const float* w, int64_t n, int32_t d, float* u, int64_t ldu, void* stream);
/* stat += sum x^2 (before scaling); x *= alpha   (turns d(logit)/d(input) into d(penalty)/d(that)) */
PHC_API int phc_scale_sumsq(float* x, int64_t ld, int64_t n, int32_t d, float alpha, float* stat, void* stream);
/* y += alpha*x on a strided block; optional stat += sum x^2   (logit regulariser / weight decay, :745-747,:771-775) */
PHC_API int phc_axpy2d(const float* x, int64_t ldx, float* y, int64_t ldy, int64_t rows, int32_t cols, float alpha,
               float* sumsq_stat, void* stream);
/* HumanoidImMCP.step action mixing (phc/env/tasks/humanoid_im_mcp.py:79-82): out[n,a] = sum_k weights[n,k] * prim_k[n,a];
 * the K primitive outputs are matrices with row stride ldp placed prim_stride floats apart.
 * discrete != 0: weights are replaced by the one-hot of their arg-max (discrete_moe, humanoid_im_mcp.py:70-72). */
PHC_API int phc_mcp_combine(const float* weights, int64_t ldw, const float* prim, int64_t ldp, int64_t prim_stride, int64_t n,
                    int32_t K, int32_t A, int32_t discrete, float* out, int64_t ldo, void* stream);
/* backward of the activation that ends the MCP composer (amp_network_mcp_builder.py:57-63, ending_act: True):
 * act = PHC_ACT_RELU: dy *= (aux > 0), aux = the composer output; act = PHC_ACT_SILU: dy *= silu'(aux), aux = pre-activation */
PHC_API int phc_act_backward(float* dy, int64_t ldd, const float* aux, int64_t ldaux, int64_t n, int32_t d, int32_t act, void* stream);
/* out[0] = sum g^2 (fp64) over the flat gradient bucket */
PHC_API int phc_grad_sumsq(const float* g, int64_t n, double* out, void* stream);
/* nn.utils.clip_grad_norm_(max_norm) (amp_agent.py:670,677) + torch.optim.Adam step (common_agent.py:67) fused over
 * the flat bucket; grad_scale = 1/world_size after the sum all-reduce; max_norm <= 0 disables clipping. */
PHC_API int phc_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n,
                  const double* grad_sumsq, float grad_scale, float max_norm, float lr, float beta1, float beta2, float eps,
                  int64_t step, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PHC_B200_H_ */
