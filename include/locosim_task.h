/*
 * TaskSpec wire format: everything of LocoEnv.step()/reset() that is not mj_step, flattened.
 *
 * Replaces (reference file:line):
 *   observation gather   mushroom ObservationHelper._build_obs driven by the env's observation_spec
 *                        (unitreeA1.py:778-835, base_humanoid.py:292-391, atlas.py:485-562, talos.py:523-598)
 *                        + LocoEnv._create_observation (base.py:584-604; unitreeA1.py:454-476,722-753)
 *   termination          LocoEnv.is_absorbing -> _has_fallen (base.py:243-255; unitreeA1.py:503-536;
 *                        base_humanoid.py:129-180; atlas.py:366-418; talos.py:356-405)
 *   reward               utils/reward.py:34-117 via LocoEnv.reward (base.py:170-176)
 *   action scaling       LocoEnv._preprocess_action (base.py:606-621, 121-126)
 *   foot forces          LocoEnv._simulation_post_step / _get_ground_forces / _create_observation with use_foot_forces
 *                        (base.py:94-98,584-604,623-631,656-679)
 *   reset                LocoEnv.reset/setup/set_sim_state + Trajectory.reset_trajectory
 *                        (base.py:178-241,478-497; utils/trajectory.py:236-273)
 *
 * Two blobs (int32 / float64): header then arrays, tightly packed, in the order below.
 */
#ifndef LOCOSIM_TASK_H
#define LOCOSIM_TASK_H

#define LOCOSIM_TASK_MAGIC 0x5441534B
#define LOCOSIM_TASK_VERSION 4

enum {
  TKI_MAGIC = 0, TKI_VERSION, TKI_OBS_DIM, TKI_N_DONE, TKI_REWARD_TYPE, TKI_N_SUBSTEPS, TKI_N_TRAJ, TKI_TRAJ_LEN,
  TKI_N_GOAL, TKI_RECENTER0, TKI_RECENTER1, TKI_REWARD_I0, TKI_REWARD_I1, TKI_REWARD_I2, TKI_REWARD_I3,
  TKI_USE_ABSORBING,
  TKI_N_GRF,      /* number of foot-force groups (0: use_foot_forces off) */
  TKI_N_GRF_GEOM, /* length of the grf_group array (= ngeom of the compiled model, 0 if n_grf == 0) */
  TKI_ROT_Q,      /* setup_random_rot (unitreeA1.py:270-285, utils/math.py:5-31): qpos index of the yaw joint, -1 = off */
  TKI_ROT_VX,     /*   dof index of the root x velocity */
  TKI_ROT_VY,     /*   dof index of the root y velocity: at every reset yaw += a (wrapped to [-pi,pi)), (vx,vy) rotated by a ~ U[0,2pi) */
  TKI_RESERVED1, TKI_RESERVED2, TKI_RESERVED3,
  TKI_HEADER_LEN = 24
};
/* int arrays after the header: obs_src_type[obs_dim], obs_src_idx[obs_dim], done_obs_idx[n_done],
 *                                  act_idx[nu]  (data.ctrl[act_idx[k]] = action[k]*act_delta[k] + act_mean[k]; mushroom's
 *                                  `self._data.ctrl[self._action_indices] = action`),
 *                                  grf_group[n_grf_geom]: per geom -1 = none, k < n_grf = member of foot group k,
 *                                  LS_GRF_FLOOR = floor (collision_groups of the env; base.py:667-679, unitreeA1.py:223-227,551-562) */

enum { TKR_REWARD_P0 = 0, TKR_REWARD_P1,
       TKR_TRACK_WP, TKR_TRACK_KP, TKR_TRACK_WV, TKR_TRACK_KV,   /* LS_REWARD_TRACKING weights / scales */
       TKR_HEADER_LEN = 8 };
/* real arrays after the header: act_mean[nu], act_delta[nu], done_lo[n_done], done_hi[n_done],
 *                               traj_table[n_traj][traj_len][nq + nv + n_goal]                      */

/* obs_src_type */
enum { LS_OBS_QPOS = 0, LS_OBS_QVEL = 1, LS_OBS_GOAL = 2,
       LS_OBS_GRF = 3 /* idx = 3*group + component: mean over the sub-steps of the control step of the contact-frame force
                         (normal, tangent1, tangent2: mj_contactForce) of the FIRST floor contact of the group, / 1000
                         (base.py:94-98,596-599,623-631; 0 in the reset observation) */ };
/* LS_OBS_PARAM = 4: idx-th user feature of the env's parameter-pool row (multi-model envs: the carried weight's mass,
   base_robot_humanoid.py:119-123; the row layout ends with meaninertia, LS_POOL_USER user floats, padding) */
#define LS_OBS_PARAM 4
#define LS_POOL_USER 4
#define LS_GRF_FLOOR 127
#define LS_MAX_GRF 4
/* reward types (utils/reward.py) */
enum {
  LS_REWARD_NONE = 0,            /* NoReward :34 */
  LS_REWARD_TARGET_VELOCITY = 1, /* TargetVelocityReward :66   exp(-(prev_obs[i0]-p0)^2) */
  LS_REWARD_VELOCITY_VECTOR = 2, /* VelocityVectorReward :100  exp(-5*|v_xy - goal*[cos,sin]|), i0=x i1=y i2=cos idx i3=goal idx */
  LS_REWARD_POS = 3,             /* PosReward :44  prev_obs[i0] */
  /* Mocap-tracking reward (BASELINE config 3 "imitation reward vs mocap dataset"). NOT in the reference (none of its six
   * rewards reads the trajectory, SURVEY F7): this package's own spec, DeepMimic-style. Every env carries a trajectory
   * cursor (traj, sample), set by each (auto-)reset to the sampled reset row and advanced by one sample per control
   * step (clamped at the last sample; with the engine setting end_of_trajectory, include/locosim.h locosim_set_time_limit,
   * the cursor advances under every reward type and the step that puts it on the last sample truncates the episode, so no
   * two steps of an episode are rewarded against the same row). With P / V = the observation entries gathered from qpos / qvel,
   *   r = wp * exp(-kp * sum_{k in P} (obs[k] - ref[k])^2) + wv * exp(-kv * sum_{k in V} (obs[k] - ref[k])^2),
   * evaluated on the observation AFTER the step against the table row at the advanced cursor (the reward of the step
   * that reached it; the observation's root x / y are not part of it). */
  LS_REWARD_TRACKING = 4
};

#endif
