/*
 * locosim C-ABI: the drop-in boundary of the H100 (sm_90a) batched LocoEnv.step() engine.
 *
 * The reference has no FFI: its hot path is reached through the Python class hierarchy
 *   LocoEnv.step/reset                      /root/reference/loco_mujoco/environments/base.py:25,178-203 (step inherited
 *                                           from mushroom_rl MultiMuJoCo -> mujoco.mj_step, parameters base.py:32-33,109-111)
 *   GymnasiumWrapper.step/reset             /root/reference/loco_mujoco/environments/gymnasium.py:47-77
 * Each entry point below names the reference call it replaces. The Python facade
 * (loco_mujoco_b200/environments/base.py) binds these with ctypes; INTEGRATION.md shows the stub a maintainer of the
 * reference would add.
 *
 * Conventions: plain pointers + sizes, no C++/torch types. All `d_*` pointers are DEVICE pointers owned by the
 * caller (e.g. torch.cuda tensors), row-major, env-major ([n_envs, dim]). All work is enqueued on `stream`
 * (a cudaStream_t passed as void*; NULL = default stream); calls are CUDA-graph capturable; no allocation happens
 * in step/reset. Return value: 0 = OK, non-zero = error, message via locosim_last_error(). Never throws.
 * One handle per device; calls on one handle must be externally serialised.
 */
#ifndef LOCOSIM_H
#define LOCOSIM_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct locosim_handle locosim_t;

/* Replaces LocoEnv.__init__ -> MultiMuJoCo.__init__ (model compile + MjData) and load_trajectory
 * (base.py:31-143,145-168).  `model_*`: ModelPack blobs (include/locosim_modelpack.h); `task_*`: TaskSpec blobs
 * (include/locosim_task.h).  env_id_offset: global index of this shard's first env (multi-GPU sharding keeps the
 * per-env random streams identical to the single-GPU run). */
int locosim_create(const int32_t* model_ints, int n_model_ints, const double* model_reals, int n_model_reals,
                   const int32_t* task_ints, int n_task_ints, const double* task_reals, int n_task_reals,
                   int n_envs, int device, uint64_t seed, int64_t env_id_offset, locosim_t** out);
void locosim_destroy(locosim_t* h);
const char* locosim_last_error(const locosim_t* h);   /* h may be NULL: error of the last failed create */

int locosim_num_envs(const locosim_t* h);
int locosim_obs_dim(const locosim_t* h);
int locosim_action_dim(const locosim_t* h);
int locosim_nq(const locosim_t* h);

/* Newton-solver controls of the fp32 engine (defaults: tolerance 1e-5, ls_tolerance 0.1, max_iter 20, ls_iter 16) */
int locosim_set_solver(locosim_t* h, float tolerance, float ls_tolerance, int max_iter, int ls_iter);

/* Replaces LocoEnv.reset() (base.py:178-203 -> setup :205-241 -> Trajectory.reset_trajectory trajectory.py:236-273
 * -> set_sim_state :478-497).  d_mask: uint8 [n_envs] (NULL = all).  Draws (traj, sample) per env from the
 * counter-based stream unless d_traj_no / d_step_no (int32 [n_envs], may be NULL) pin them.  Writes the reset
 * observation to d_obs ([n_envs, obs_dim], may be NULL). */
int locosim_reset(locosim_t* h, const uint8_t* d_mask, const int32_t* d_traj_no, const int32_t* d_step_no, float* d_obs,
                  void* stream);
/* Same, with the parameter-pool row (= the model of a multi-model env, `np.random.randint(0, len(self._models))` in
 * base.py:187-191) pinned per env as well: d_pool_row int32 [n_envs] or NULL (draw from the counter-based stream). */
int locosim_reset_rows(locosim_t* h, const uint8_t* d_mask, const int32_t* d_traj_no, const int32_t* d_step_no,
                       const int32_t* d_pool_row, float* d_obs, void* stream);

/* Replaces LocoEnv.step(action) (mushroom MuJoCo.step: _preprocess_action base.py:606-621, n_substeps x mj_step,
 * _create_observation :584-604, is_absorbing :243-255, reward :170-176) for every env of the batch, followed by an
 * in-kernel auto-reset of the envs that terminated.
 *   d_action   [n_envs, action_dim] in [-1, 1]
 *   d_obs      [n_envs, obs_dim]   observation after the step (the terminal observation for envs with done=1)
 *   d_reward   [n_envs]
 *   d_done     [n_envs] uint8      bit 0 = absorbing (has_fallen, or non-finite state); bit 1 (value 2) = truncated by a time
 *                                  limit (locosim_set_time_limit; never set while both limits are off)
 *   d_next_obs [n_envs, obs_dim]   observation to act on next (== d_obs unless done, then the reset observation); may be NULL
 * auto_reset: 0 leaves terminated envs in their terminal state (caller resets with locosim_reset); truncated envs are
 * auto-reset exactly like terminated ones. */
int locosim_step(locosim_t* h, const float* d_action, float* d_obs, float* d_reward, uint8_t* d_done, float* d_next_obs,
                 int auto_reset, void* stream);

/* State access (LocoEnv.set_sim_state base.py:478-497 / data.qpos, data.qvel). fp32 [n_envs, nq]. */
int locosim_get_state(locosim_t* h, float* d_qpos, float* d_qvel, float* d_qacc_warmstart, void* stream);
int locosim_set_state(locosim_t* h, const float* d_qpos, const float* d_qvel, const float* d_qacc_warmstart, void* stream);

/* setup_random_rot in the drop-in single-env mode (unitreeA1.py:270-285: angle = np.random.uniform(0, 2 pi) from the legacy
 * numpy stream): rotation angles for the NEXT locosim_reset* call only, d_angle fp32 [n_envs] (NULL: the engine's own
 * counter-based draw, which is also what in-kernel auto-resets use). Requires a TaskSpec with TKI_ROT_* set. */
int locosim_set_reset_rotation(locosim_t* h, const float* d_angle);

/* Trajectory cursor of every env (traj * traj_len + sample; LS_REWARD_TRACKING and end_of_trajectory, include/locosim_task.h).
 * int32 [n_envs]. */
int locosim_get_cursor(locosim_t* h, int32_t* d_out, void* stream);

/* Time limit: ends episodes that neither fall nor diverge. The reference leaves this to its consumer (mushroom Core enforces
 * MDPInfo.horizon, and resets when Trajectory.get_next_sample() returns None: utils/trajectory.py:311-323, base.py:365-368);
 * a batched loop relies on the in-kernel auto-reset, so the engine enforces it. An engine setting like locosim_set_solver
 * (not part of the TaskSpec: one compiled task serves training with and evaluation without a limit). 0, 0 = off = the state
 * after locosim_create; negative values are an error. Takes effect from the next locosim_step.
 *
 * Episode length = control steps since the env's last reset of any kind (locosim_reset*, in-kernel auto-reset);
 * locosim_set_state does not restart it. Two independent limits:
 *   max_episode_steps = H > 0: the episode is truncated by the control step that makes its length reach H.
 *   end_of_trajectory = 1:     the trajectory cursor advances by one sample per control step under EVERY reward type (one
 *       advance per step; LS_REWARD_TRACKING compares against the row at the advanced cursor as always), and the episode
 *       is truncated by the step after which the cursor stands on the LAST sample of its trajectory: the step for which
 *       get_next_sample() would next return None, i.e. the last step whose tracking reward has a table row of its own.
 *       An episode reset to sample s of a trajectory of traj_len samples is therefore truncated by its step number
 *       traj_len - 1 - s (s = traj_len - 3: second step, s = traj_len - 2: first step). An episode reset ONTO the last
 *       sample cannot advance: its first step is truncated and the cursor stays where it is.
 *       With the option off the cursor moves under LS_REWARD_TRACKING only and is clamped at the last sample.
 * Absorbing wins: a step that is terminal and at a limit reports bit 0 only. With auto_reset = 1 a truncated env is reset in
 * the same step like a fallen one (d_obs = the final observation of the old episode, d_next_obs = the reset observation;
 * episode counter, pool row, goal, rotation, cursor and LOCOSIM_KEY_RESET as for any auto-reset). With auto_reset = 0 bit 1
 * is reported on that step and on every later step until the caller resets the env; nothing else changes. */
int locosim_set_time_limit(locosim_t* h, int max_episode_steps, int end_of_trajectory);

/* Per-episode statistics, kept per env on the device whether or not a limit is set: d_len int32 / d_ret fp32 = control steps
 * and sum of the rewards locosim_step wrote (fp32, in step order) of the RUNNING episode (both 0 after a reset); d_last_len /
 * d_last_ret = the same two of the env's last FINISHED episode (finished = a step reported absorbing or truncated; 0 before
 * the first one; an env that stays finished under auto_reset = 0 rewrites them every step). Rewards evaluated outside the
 * engine (LS_REWARD_NONE, the Python facade's reward_type="custom") count as the 0 the engine writes. Each [n_envs], each
 * may be NULL; stream-ordered copies like locosim_get_cursor. */
int locosim_get_episode_stats(locosim_t* h, int32_t* d_len, float* d_ret, int32_t* d_last_len, float* d_last_ret, void* stream);

/* Bodies of the compiled model, the world (body 0) included: the row length of the xfrc_applied buffer below is 6 * nbody.
 * Body indices are those of the compiled model (fuse_static merges static bodies into their parents). */
int locosim_nbody(const locosim_t* h);

/* Applied forces, MuJoCo 2.3.7's mjData.xfrc_applied / qfrc_applied (how a loco-mujoco user pushes a robot through
 * env._data): caller-owned DEVICE buffers, registered once and read by every later locosim_step.
 *   d_xfrc fp32 [n_envs, nbody, 6]: per body a force (3) then a torque (3), world coordinates, applied at the body's centre
 *          of mass (xipos), as mj_applyFT does. Row 0 (the world) is ignored.
 *   d_qfrc fp32 [n_envs, nq]:       generalised forces.
 * Either may be NULL; NULL, NULL = off = the state after locosim_create (nothing is read then, and no output changes by a bit).
 * Semantics of mj_fwdAcceleration + mj_xfrcAccumulate: qfrc_smooth = passive - bias + actuator + qfrc_applied
 * + sum over bodies of J_b^T xfrc_applied[b], in EVERY dynamics evaluation with that evaluation's kinematics (Euler: once per
 * sub-step; RK4: each of the four stages); the constraint solver sees them through qacc_smooth.
 * They last until the caller changes them: the engine only writes zeros, into the rows of every env it resets (locosim_reset*
 * for the masked envs, the in-kernel auto-reset for the envs it resets), as mj_resetData does; locosim_set_state leaves them
 * alone. So the buffers must stay valid and writable while registered. An engine setting like locosim_set_time_limit (not
 * part of the TaskSpec); takes effect from the next locosim_step. The pointers are engine state, not per-call values: register
 * them outside of stream capture (before cudaStreamBeginCapture); a captured step then reads whatever the buffers hold when
 * it is replayed. */
int locosim_set_applied_forces(locosim_t* h, float* d_xfrc, float* d_qfrc);

/* Terrain (height field) origin per env. A model packed with a terrain (include/locosim_modelpack.h: UnitreeA1 only; any other
 * model with a terrain is refused at create) runs on the kernel configuration CfgEllEulerTerrain. Semantics, MuJoCo 2.3.7's
 * hfield geom and mjc_ConvexHField as this project defines them:
 *   Shape: nrow x ncol samples (nrow, ncol >= 2), size = (rx, ry, elevation, base). Sample (r, c) sits at
 *     x = c * 2 rx / (ncol - 1) - rx, y = r * 2 ry / (nrow - 1) - ry, z = data[r * ncol + c] * elevation in the geom's frame
 *     (data normalised to [0, 1], as MuJoCo's compiler stores it); the solid reaches down to z = -base. One field per model,
 *     unrotated (a geom quaternion other than identity is refused).
 *   Prisms: each cell (r, c) is split into two triangles, extruded down to -base: triangle 0 = grid points (c, r), (c, r+1),
 *     (c+1, r), triangle 1 = (c, r+1), (c+1, r), (c+1, r+1), i.e. the diagonal from (c+1, r) to (c, r+1), the triangles of
 *     MuJoCo's strip builder in mjc_ConvexHField as this project restates it (MuJoCo's source could not be checked here:
 *     this is THIS PROJECT'S DEFINITION, used by collision, the fp64 reference and the ray caster alike). A prism's six
 *     vertices are ordered bottom (z = -base) then top, each in the triangle's order; its support is the first maximum of
 *     the six, its centre (MPR's first portal point) their mean.
 *   Collision of the terrain with a robot geom g (sphere, capsule, cylinder or box): g is expressed in the field's frame; its
 *     bounding box comes from its support along +-x, +-y, +-z; the pair ends when that box, grown by the pair's margin,
 *     misses the field's box [-rx, rx] x [-ry, ry] x [-base, elevation]. The cell range is floor / ceil of the grown box's
 *     grid coordinates, clamped to the grid. Prisms are taken in (row, column, triangle) order; one whose three top points
 *     all lie below (lowest point of g) - margin is skipped; every other one runs MPR (the engine's mjc_Convex) with each
 *     side inflated by margin / 2, and each one that penetrates gives one contact: dist = margin - depth, the MPR normal
 *     (from the terrain into g) and position, as for every convex pair. At most 50 contacts per pair (mjMAXCONPAIR); the
 *     margin handling is this project's definition too.
 *   Contact parameters: the terrain geom carries the floor geom's contype / conaffinity, friction, condim, solref, solimp,
 *     solmix, priority, margin and gap; it is paired with exactly the geoms the floor is paired with, and it is geom1 of
 *     those pairs. The terrain pairs come after every other pair. The floor plane stays: a terrain above the floor hides it,
 *     a pit can reach down to it.
 *   Origin: env i sees the field translated by (-origin[i][0], -origin[i][1], 0): origin[i] is the terrain point (x, y) under
 *     env i's world origin, its reset spot. Resets are unchanged (root x / y zeroed, root z from the dataset): it is the
 *     terrain's job to be flat at height 0 under every spawn point (loco_mujoco_b200/terrain.py builds such fields). The
 *     termination test is unchanged too: UnitreeA1's q_trunk_tz > -0.24 ends an episode in a pit deeper than 0.24 m.
 * d_origin: caller-owned fp32 [n_envs, 2], read by every later step and on-demand query (locosim_inverse, locosim_forward,
 * locosim_dynamics_terms, ...). NULL = all zeros = the state after locosim_create. Like the applied-force buffers, the origin is
 * not part of a saved state row: index it with the same rows. Register outside of stream capture, like
 * locosim_set_applied_forces. Refused on a handle without a terrain. locosim_create_dataset_inverse evaluates dataset rows, not
 * envs: they take the zero origin.
 *   Rays (locosim_ray): the terrain is a static geom of the world body (LS_RAY_STATIC; excluded with exclude_body 0), cast
 *     in env i's translated frame as mj_rayHfield: the top triangles (the diagonal above), the four sides up to the
 *     surface along the edge, and the base; the first hit of any of them, with its outward normal. */
int locosim_set_terrain_origin(locosim_t* h, float* d_origin);

/* Body outputs, MuJoCo's per-body kinematics (what a loco-mujoco user reads from env._data: xpos, xquat, body velocities):
 * caller-owned DEVICE buffers, each fp32 [n_envs, nbody, LS_BODY_DIM]. Per body (row) 13 values:
 *   xpos (3)  world position of the body frame
 *   xquat (4) orientation of the body frame, w x y z
 *   angular velocity (3), then linear velocity (3) of the body-frame origin xpos, both in world coordinates: the result of
 *             mj_objectVelocity(m, d, mjOBJ_XBODY, b, res, 0), in its order. The point is the body-frame origin, NOT the centre
 *             of mass (xipos) that xfrc_applied acts at.
 * Row 0 (the world) is (0,0,0, 1,0,0,0, 0,0,0, 0,0,0). Body indices are those of the compiled model, as for xfrc_applied.
 * The values describe the state they are written for: mj_kinematics + mj_comPos + mj_comVel evaluated on that state's qpos /
 * qvel, i.e. what mj_forward on that state gives. This differs from MuJoCo's mjData after mj_step, whose kinematic fields
 * still describe the start of the last sub-step (after RK4: its last stage); here they describe the same state as the
 * observation.
 *   d_body:      written by every locosim_step for the state d_obs describes: for an env that ended, its terminal state
 *                (before the auto-reset); for a non-finite env all zeros, as its observation.
 *   d_next_body: always the state locosim_get_state returns: written by locosim_step after the auto-reset (rows of envs not
 *                reset equal d_body bit for bit), by locosim_reset* for the masked envs and by locosim_set_state for every env.
 * While either is registered, locosim_step enqueues one more kernel after the step (the rows of envs it resets are written
 * by the step kernel before the reset, every other row from the stored state), and locosim_reset* / locosim_set_state one
 * kernel each when d_next_body is registered. Either may be NULL; NULL, NULL = off = the state after locosim_create (nothing
 * is written or launched then, and no other output changes by a bit; with buffers registered no other output changes by a
 * bit either). Register outside of stream capture, like locosim_set_applied_forces.
 * CUDA graphs: whether the extra kernel is part of a step is decided when the step is enqueued (or captured). A graph captured
 * while something is registered writes, at each replay, into whatever non-NULL buffers are registered then (a later
 * registration of other buffers is picked up; NULL, NULL makes its extra kernel write nothing). A graph captured while
 * NOTHING was registered never writes d_next_body, nor d_body of envs it does not reset: after turning the feature on,
 * capture the step again. (Each registration clears the engine's per-env reset marks, and under auto_reset the rows an
 * eager or re-captured step writes never depend on what such a stale graph did.) */
#define LS_BODY_DIM 13
int locosim_set_body_outputs(locosim_t* h, float* d_body, float* d_next_body);

/* Contact outputs, MuJoCo's contact forces summed per body (what a loco-mujoco user computes with mj_contactForce over
 * env._data.contact): a caller-owned DEVICE buffer d_contact, fp32 [n_envs, nbody, LS_CONTACT_DIM]. Rows are the compiled
 * model's body indices, as for xfrc_applied and the body outputs. Per body 6 values, the wrench exerted ON the body BY all of
 * its contacts:
 *   force (3)  world coordinates
 *   torque (3) world coordinates, about the body-frame origin xpos (the point of the body outputs' linear velocity). NOT the
 *              centre of mass, and NOT the subtree_com convention of MuJoCo's cfrc_ext.
 * Per contact, f = the contact-frame force of mj_contactForce (elliptic cones: the dim constraint forces; pyramidal cones:
 * mju_decodePyramid; dim 1, 3, 4 and 6), and with the frame rows n, t1, t2 (n points from geom1 to geom2):
 *   F = f0 n + f1 t1 + f2 t2,  T = f3 n + f4 t1 + f5 t2 (the components past dim are zero).
 * The contact adds +F and (pos - xpos[b2]) x F + T to geom2's body b2, and -F and -((pos - xpos[b1]) x F + T) to geom1's body
 * b1 (the signs of mj_rnePostConstraint). A self contact therefore appears in two rows with opposite signs. Row 0 (the world)
 * is all zeros.
 * Time window: the MEAN over the control step's sub-steps; each sub-step contributes the contact list, xpos and constraint
 * forces of its last dynamics evaluation (Euler: its only one; RK4: its fourth stage), the window and evaluation of the
 * use_foot_forces observation. This differs from MuJoCo's mjData after mj_step, which holds the last sub-step only. Contacts
 * dropped by the per-env cap of the constraint set (DESIGN.md section 7) are not in the sum.
 * Written by every locosim_step for every env it advances: the row describes the step that produced d_obs (for an env that
 * ended and was auto-reset: its terminal step; for a non-finite env all zeros, as its observation). Not written by
 * locosim_reset* or locosim_set_state. NULL = off = the state after locosim_create: nothing is written, and no other output
 * changes by a bit; with the buffer registered no other output changes by a bit either. Register outside of stream capture,
 * like locosim_set_applied_forces.
 * CUDA graphs: the step kernels read the pointer from engine state on the device when they run, and no kernel is added. A
 * step captured BEFORE the registration therefore writes the buffer when it is replayed after it (unlike the body outputs),
 * and registering NULL stops a captured step writing. */
#define LS_CONTACT_DIM 6
int locosim_set_contact_outputs(locosim_t* h, float* d_contact);

/* Per-dof outputs, MuJoCo's mjData.qfrc_actuator / qfrc_constraint / qacc (what a loco-mujoco user reads from env._data for
 * torque, joint-limit and acceleration penalties): a caller-owned DEVICE buffer d_dof, fp32 [n_envs, nq, LS_DOF_DIM]. Every
 * in-scope model has nq == nv (hinge and slide joints only), so rows are dof indices: the qvel layout of locosim_get_state
 * and of qfrc_applied. Per dof 3 values:
 *   0 qfrc_actuator    sum over the actuators on the dof of gear * force, the force of mj_fwdActuation: ctrl clamped to
 *                      ctrlrange, gain * ctrl + bias0 + bias1 * qpos + bias2 * qvel at the evaluation's state, clamped to
 *                      forcerange
 *   1 qfrc_constraint  J^T efc_force at the solver's final qacc, as mj_fwdConstraint leaves it
 *   2 qacc             the constrained acceleration of mj_forward. For the Euler integrator this is NOT the solve with
 *                      implicit joint damping that the integrator advances with (which MuJoCo also keeps out of d->qacc).
 *                      locosim_inverse below is the continuous-time inverse of this qacc; MuJoCo 3's discrete-time inverse
 *                      (mjENBL_INVDISCRETE), which would invert the implicit-damping solve, is not built.
 * Time window: the MEAN over the control step's sub-steps; each sub-step contributes its last dynamics evaluation (Euler: its
 * only one; RK4: its fourth stage), the window of the contact outputs. This differs from MuJoCo's mjData after mj_step, which
 * holds the last sub-step only, evaluated at that sub-step's START state (RK4: its first stage).
 * Written by every locosim_step for every env it advances: the row describes the step that produced d_obs (for an env that
 * ended and was auto-reset: its terminal step; for a non-finite env all zeros, as its observation). Not written by
 * locosim_reset* or locosim_set_state. NULL = off = the state after locosim_create: nothing is written, and no other output
 * changes by a bit; with the buffer registered no other output changes by a bit either. Register outside of stream capture.
 * CUDA graphs: as for the contact outputs, the step kernels read the pointer from engine state on the device when they run
 * and no kernel is added, so a step captured BEFORE the registration writes the buffer when it is replayed after it. */
#define LS_DOF_DIM 3
int locosim_set_dof_outputs(locosim_t* h, float* d_dof);

/* Contact list, MuJoCo's d->contact[:d->ncon] with each contact's mj_contactForce (what a loco-mujoco user reads from
 * env._data.contact after env.step(): support polygons, ZMP and support-margin terms, per-corner forces of box feet,
 * penetration depth, per-pair self-collision penalties). Three caller-owned DEVICE buffers, MAXC = locosim_max_contacts(h)
 * (the configuration's per-env contact cap, 16 in every configuration):
 *   d_ncon    int32 [n_envs]                           the number of contacts in the list
 *   d_con     fp32  [n_envs, MAXC, LS_CONLIST_DIM]     per contact, at the LS_CONLIST_* columns:
 *               DIST (1)   the signed distance (negative: penetration)
 *               POS (3)    the contact position, world frame
 *               FRAME (9)  the contact frame's rows n, t1, t2 (world frame; n points from geom1 to geom2)
 *               FORCE (6)  the contact-frame force f of mj_contactForce (normal, two tangents, torsion, two rolling;
 *                          elliptic cones: the dim constraint forces; pyramidal cones: mju_decodePyramid). The components
 *                          past dim are 0. The world-frame force is f0 n + f1 t1 + f2 t2, and it acts on geom2 (its
 *                          negative on geom1), as in the contact outputs above.
 *   d_con_id  int32 [n_envs, MAXC, LS_CONLIST_ID_DIM]  GEOM1, GEOM2 (the compiled model's geom indices), BODY1, BODY2
 *                                                     (geom_bodyid: the rows of the body and contact outputs), CONDIM (dim)
 * Rows at and past ncon are written on every step too: fp32 zeros and ids of -1, so nothing of an earlier step survives
 * and masked reductions need no clean-up.
 * Time window: the contact list of the control step's LAST sub-step at its last dynamics evaluation (Euler: the sub-step's
 * only one, at its start state; RK4: its fourth stage), and that evaluation's constraint forces. This is what MuJoCo 2.3.7's
 * mjData holds after mj_step (Euler: the mj_forward at the start of the last sub-step; RK4: mj_RungeKutta's last
 * mj_forwardSkip, whose d->contact and d->efc_force are not restored), so the rows are what the reference's user reads
 * after env.step(), up to fp32 and the cap. The contact outputs above are instead the MEAN over all sub-steps, summed per
 * body. With n_substeps = 1 the two describe the same evaluation.
 * Order: the engine's list order, the one use_foot_forces takes its "first contact" from: candidate pairs in the compiled
 * pair table's order (primitive pairs first, then the general convex (MPR) pairs, each part in model order), and within a
 * pair the narrow phase's order. The package's fp64 reference builds its list from the same table in the same order, so
 * the rows match its rows one for one while nothing is dropped (tests compare them in order). MuJoCo's own broad phase may
 * visit the pairs in another order: compare with a MuJoCo list as a set of geom pairs. Contacts the gap excludes (dist >=
 * margin - gap), which MuJoCo keeps in d->contact without a constraint, are not in the list.
 * Cap: contacts past MAXC, and those cut when their constraint rows would overflow the per-env row cap (DESIGN.md section
 * 7), are not in the list and are not counted. ncon == MAXC is the only sign that contacts may have been dropped.
 * Written by every locosim_step for every env it advances: the rows describe the step that produced d_obs (for an env that
 * ended and was auto-reset: its terminal step; for a non-finite env ncon = 0 and empty rows). Not written by locosim_reset*,
 * locosim_set_state or locosim_load_state.
 * All three buffers non-NULL turns the list on; all three NULL turns it off (the state after locosim_create): nothing is
 * written then, and no other output changes by a bit. With the buffers registered no other output changes by a bit either.
 * Any other combination, and buffers that overlap, are refused. Register outside of stream capture.
 * CUDA graphs: as for the contact outputs, the step kernels read the pointers from engine state on the device when they run
 * and no kernel is added, so a step captured BEFORE the registration writes the buffers when it is replayed after it, and
 * registering NULLs stops a captured step writing. */
#define LS_CONLIST_DIM 19
#define LS_CONLIST_DIST 0
#define LS_CONLIST_POS 1
#define LS_CONLIST_FRAME 4
#define LS_CONLIST_FORCE 13
#define LS_CONLIST_ID_DIM 5
#define LS_CONLIST_GEOM1 0
#define LS_CONLIST_GEOM2 1
#define LS_CONLIST_BODY1 2
#define LS_CONLIST_BODY2 3
#define LS_CONLIST_CONDIM 4
int locosim_max_contacts(const locosim_t* h);
int locosim_set_contact_list_outputs(locosim_t* h, int32_t* d_ncon, float* d_con, int32_t* d_con_id);

/* Replaces LocoEnv.create_dataset() (base.py:278-312 -> utils/trajectory.py:104-151) on the device: consecutive samples of
 * every trajectory of the reset table in observation layout. d_states / d_next_states fp32 [locosim_dataset_rows, obs_dim],
 * d_last fp32 [locosim_dataset_rows] (may be NULL); absorbing is all zero in the reference and is not materialised. */
int locosim_dataset_rows(const locosim_t* h);
int locosim_create_dataset(locosim_t* h, float* d_states, float* d_next_states, float* d_last, void* stream);

/* Reference outputs: the body outputs of the mocap clip, the expert side of body-space imitation terms (end-effector and
 * centre-of-mass tracking, keypoint discriminators, foot placement). Caller-owned DEVICE buffers, each fp32
 * [n_envs, nbody, LS_BODY_DIM]; a REFERENCE ROW has the layout and body indices of the body outputs above.
 * The reference row of an env is the body outputs of the state locosim_reset_rows would give it if it were reset onto the
 * table row (traj, sample) at its cursor (locosim_get_cursor): reset_value of that row, i.e. root x / y zeroed and, under
 * setup_random_rot, the yaw shifted and root (vx, vy) rotated by the rotation angle of the env's CURRENT episode (the one its
 * last reset drew or was given by locosim_set_reset_rotation), evaluated with the env's current parameter-pool row.
 * So immediately after any reset the reference row equals d_next_body of the same env bit for bit. Positions are therefore
 * root-x/y-relative: to compare a simulated body with its reference, subtract the simulated root's x / y first, e.g.
 *   foot = body[i, b, 0:3];  foot.x -= body[i, root, 0];  foot.y -= body[i, root, 1];
 *   err  = |foot - ref[i, b, 0:3]|      (the reference root stands at x = y = 0)
 * Phase = the cursor: it advances by one sample per control step under LS_REWARD_TRACKING or end_of_trajectory
 * (locosim_set_time_limit), clamped at the last sample. With neither, the cursor stays on the reset row and so does the
 * reference (this is not refused here).
 *   d_ref:      written by every locosim_step for the state d_obs describes: for an env that ended, the cursor its terminal
 *               step reached, before the auto-reset moves the cursor (and that episode's angle and pool row); for a
 *               non-finite env all zeros, as in d_body.
 *   d_next_ref: the state to act on next: written by locosim_step after the auto-reset (rows of envs not reset equal d_ref bit
 *               for bit) and by locosim_reset* for the masked envs. locosim_set_state moves no cursor and does not write it.
 * Either may be NULL; NULL, NULL = off = the state after locosim_create: nothing is written or launched, and no other output
 * changes by a bit; with buffers registered no other output, the body outputs included, changes by a bit either. The rows are
 * written by the body outputs' kernel after the step, so the launch and CUDA-graph rules are those of the body outputs:
 * register outside of stream capture, and capture the step again after turning the feature on (a graph captured while
 * neither body nor reference outputs were registered writes neither, and its replays do not keep the per-env record the
 * terminal rows are built from; registering again rebuilds that record). Registering reads every env's current state on the
 * device and waits for it; a new parameter pool (locosim_set_param_pool) does the same. */
int locosim_set_reference_outputs(locosim_t* h, float* d_ref, float* d_next_ref);

/* The reference rows of the whole dataset, row-aligned with locosim_create_dataset: d_body / d_next_body fp32
 * [locosim_dataset_rows, nbody, LS_BODY_DIM]. Row r is the reference row of dataset row r's (traj, sample) in d_body and of
 * (traj, sample + 1) in d_next_body, with rotation angle 0 and the compiled model's own parameters (what an env runs with when
 * no parameter pool is set). Stream-ordered; the expert side of a body-space discriminator. */
int locosim_create_dataset_bodies(locosim_t* h, float* d_body, float* d_next_body, void* stream);

/* Inverse dynamics, MuJoCo 2.3.7's continuous-time mj_inverse: the generalised force that produces a given acceleration at
 * a given state, contacts included. For an env with state (qpos, qvel), its parameter-pool row and an acceleration qacc:
 *   qfrc_inverse = M(q) qacc + qfrc_bias(q, v) - qfrc_passive(q, v) - qfrc_constraint(q, v, qacc)
 * with M including dof_armature, qfrc_bias the RNE bias with gravity, qfrc_passive the joint stiffness plus the explicit
 * damping -b qvel, and qfrc_constraint = J^T efc_force, efc_force the soft-constraint force of jar = J qacc - aref (the
 * solver's map, mj_constraintUpdate): friction loss, joint limits and contacts (the configuration's cone), over the
 * contact set the state gives, with the per-env row cap of the forward dynamics. Actuator forces, qfrc_applied and
 * xfrc_applied are NOT subtracted, as in MuJoCo, so at a forward solution
 *   qfrc_inverse ~= qfrc_actuator + qfrc_applied + J^T xfrc_applied     (up to the solver's convergence: mjENBL_FWDINV)
 * and registered applied forces change no bit of the result. The integrator plays no part (continuous time).
 * A non-finite qpos, qvel or qacc of an env gives that env a row of zeros (and that state reaches no collision test).
 * The call reads the state and changes nothing else: state, warm start, counters, cursors, random streams, episode
 * statistics and every registered output stay as they were.
 *
 * locosim_inverse: every env at its stored state (what locosim_get_state returns) and its current pool row (carry tasks:
 * the carried weight's model). d_qacc, d_qfrc_inverse fp32 [n_envs, nv] DEVICE buffers in the qvel dof order of
 * locosim_get_state and qfrc_applied (every in-scope model has nq == nv); they must not overlap (refused). Stream-ordered,
 * no host synchronisation, no allocation: it can be captured in a CUDA graph (a replay reads the buffers and the state as
 * they are then). */
int locosim_inverse(locosim_t* h, const float* d_qacc, float* d_qfrc_inverse, void* stream);

/* Inverse dynamics of the whole dataset, row-aligned with locosim_create_dataset and locosim_create_dataset_bodies:
 * d_qfrc fp32 [locosim_dataset_rows, nv]. Row r, (traj, sample) -> (traj, sample + 1), is the inverse at the reset state of
 * (traj, sample) (reset_value with rotation angle 0 and the compiled model's own parameters, as the dataset's reference
 * rows) at the forward-difference acceleration of the dataset's control rate, exactly
 *   inv_dt = (float)(1.0 / ((double)timestep * n_substeps))       (timestep: the model's fp32 timestep, on the host)
 *   qacc   = (qvel[sample + 1] - qvel[sample]) * inv_dt           (fp32, qvel as reset_value gives it)
 * so that a caller can rebuild qacc bit for bit. Stream-ordered: the forces a mocap clip needs, and the residual on the
 * unactuated root dofs. */
int locosim_create_dataset_inverse(locosim_t* h, float* d_qfrc, void* stream);

/* Model-based dynamics terms of every env at its stored state (what locosim_get_state returns, the state of
 * info["next_obs"]) with its current parameter-pool row (carry tasks: the carried weight's model), in MuJoCo 2.3.7's
 * meaning. All outputs are fp32 DEVICE buffers, env-major; dofs in the qvel order of locosim_get_state (every in-scope
 * model has nq == nv), body rows in the compiled model's body indices (those of xfrc_applied and the body outputs):
 *   d_M        [n_envs, nv, nv]         mj_fullM of d->qM: dense, symmetric, dof_armature on the diagonal
 *   d_bias     [n_envs, nv]             d->qfrc_bias: mj_rne with qacc = 0 (Coriolis, centrifugal and gravity)
 *   d_passive  [n_envs, nv]             d->qfrc_passive: -stiffness (q - q_spring) - damping qvel, the term locosim_inverse
 *                                       subtracts
 *   d_com      [n_envs, LS_COM_DIM]     the whole-robot centre of mass d->subtree_com[0] (x, y, z), then the total mass; a
 *                                       carried weight is part of the robot, and both follow the env's pool row
 *   d_jac      [n_envs, nbody, 6, nv]   per body, rows 0-2 jacr and rows 3-5 jacp of mj_jacBody: the Jacobian of the
 *                                       body-frame origin xpos (NOT xipos) in world coordinates, rows in body_state's order
 *                                       (angular, then linear velocity), so jac[i, b] @ qvel[i] = body_state[i, b, 7:13];
 *                                       body 0 (the world) is all zeros. xfrc_applied acts at xipos, so J^T F with this
 *                                       Jacobian is NOT the generalised force of an xfrc_applied force.
 *   d_jac_com  [n_envs, 3, nv]          mj_jacSubtreeCom of the whole robot: d(com) / dq, i.e. com velocity = jac_com qvel
 * Any output may be NULL; with all six NULL the call launches nothing and returns 0. Overlapping outputs are refused.
 * A non-finite qpos or qvel of an env gives that env zero rows in every output. The call reads the state and changes
 * nothing else: state, warm start, counters, cursors, random streams, episode statistics and every registered output stay
 * as they were. Stream-ordered, no host synchronisation, no allocation: it can be captured in a CUDA graph (a replay reads
 * the state as it is then). */
#define LS_COM_DIM 4
int locosim_dynamics_terms(locosim_t* h, float* d_M, float* d_bias, float* d_passive, float* d_com, float* d_jac,
                           float* d_jac_com, void* stream);

/* Forward dynamics under a given action, without advancing the env: one MuJoCo 2.3.7 mj_forward per env, followed by
 * mj_rnePostConstraint. Every env is evaluated
 *   - at its stored state (what locosim_get_state returns), with its stored qacc_warmstart as the Newton warm start;
 *   - with its current parameter-pool row (carry tasks: the carried weight's model);
 *   - with ctrl from d_action [n_envs, action_dim] exactly as locosim_step computes it (action * act_delta + act_mean into
 *     act_idx; position mode included);
 *   - with the registered xfrc_applied / qfrc_applied, read as a step reads them;
 *   - with the solver settings of locosim_set_solver.
 * The integrator plays no part: for Euler with joint damping, qacc is the explicit mj_forward one, as in the dof outputs.
 * All outputs are fp32 DEVICE buffers, env-major; dofs in the qvel order, body rows in the compiled model's body indices:
 *   d_dof       [n_envs, nv, LS_DOF_DIM]          the dof outputs' layout and meaning (qfrc_actuator, qfrc_constraint,
 *                                                 qacc) for this single evaluation, not a sub-step mean
 *   d_body_acc  [n_envs, nbody, LS_BODY_ACC_DIM]  per body the angular acceleration (3), then the linear acceleration of the
 *                                                 body-frame origin xpos MINUS gravity (3), world frame:
 *                                                 mj_objectAcceleration(m, d, mjOBJ_XBODY, b, res, 0). The angular part is
 *                                                 d/dt body_state[..., 7:10], the linear part d^2 xpos / dt^2 - gravity, so a
 *                                                 body resting on the floor reads (0, 0, +9.81) and a free-falling one 0 (an
 *                                                 accelerometer's reading). Row 0 is (0, 0, 0, -gravity), as d->cacc[0].
 *   d_cfrc_int  [n_envs, nbody, LS_CONTACT_DIM]   force (3), then torque about xpos (3), world frame: the wrench body b's
 *                                                 parent exerts on b through the joints between them (d->cfrc_int[b] moved
 *                                                 from subtree_com to xpos, force first as in the contact outputs). Row 0 is 0.
 *   d_cfrc_ext  [n_envs, nbody, LS_CONTACT_DIM]   the same layout: the external wrench on b, its contacts (the contact
 *                                                 outputs' per-contact definition over this evaluation's contact list;
 *                                                 contacts past the per-env cap are not in it) plus xfrc_applied[b] moved from
 *                                                 xipos to xpos (d->cfrc_ext). Row 0 is 0.
 * d_action is required; any output may be NULL, and with all four NULL the call launches nothing and returns 0. Outputs
 * that overlap each other or d_action are refused. A non-finite qpos, qvel or action of an env gives that env zero rows.
 * The call changes nothing: state, warm start, counters, cursors, random streams, episode statistics, every registered
 * output and the dof outputs' actuator scratch stay as they were, so a step after it is bit-identical to the same step
 * without it. Stream-ordered, no host synchronisation, no allocation: it can be captured in a CUDA graph (a replay reads the
 * action and the state as they are then). */
#define LS_BODY_ACC_DIM 6
int locosim_forward(locosim_t* h, const float* d_action, float* d_dof, float* d_body_acc, float* d_cfrc_int,
                    float* d_cfrc_ext, void* stream);

/* Saved simulation states, MuJoCo's mj_copyData for a batch: every env's whole state as one int32 row of
 * locosim_state_words() words on the device, to be loaded back into the same env or into any other env of a handle with the
 * same layout tag (forks for sampling-based MPC, reset-to-state curricula, replays).
 *
 * Row layout (the words are fp32 bits where the field is fp32; nv = locosim_nq, D = locosim_obs_dim):
 *   LS_STATE_TAG      2 words: LS_STATE_VERSION, then a fingerprint of nv, nbody, obs_dim, n_goal, n_traj and traj_len
 *                     computed when the handle is created. Two handles of one task (shards, MixedBatch members) share it.
 *   LS_STATE_EPISODE  the reset counter: the number of the env's next reset in its counter-based random stream
 *   LS_STATE_DR_ROW   the parameter-pool row (domain-randomisation draw; carry tasks: the carried weight)
 *   LS_STATE_CURSOR   the trajectory cursor traj * traj_len + sample (locosim_get_cursor)
 *   LS_STATE_ANGLE    fp32: the setup_random_rot angle of the running episode (0 without the option)
 *   LS_STATE_EP       4 words: length, return (fp32), last length, last return (fp32) (locosim_get_episode_stats)
 *   LS_STATE_GOAL     4 words (fp32): the goal features (locosim_set_goal)
 *   LS_STATE_QPOS(nv), LS_STATE_QVEL(nv), LS_STATE_WARMSTART(nv)   nv words each (fp32): locosim_get_state
 *   LS_STATE_OBS(nv)  D words (fp32): the observation the env acts on next
 *   then zeros up to LS_STATE_WORDS(nv, D), a multiple of 4.
 *
 * locosim_save_state writes one row per env into d_state int32 [n_envs, W]. d_obs fp32 [n_envs, obs_dim] is required: the
 * observation the env acts on next, i.e. a step's d_next_obs or a reset's d_obs. (The foot-force part of an observation is
 * the mean over the last step's sub-steps, which the engine does not keep after the step.)
 *
 * locosim_load_state: env i takes row d_row[i] of the n_rows rows of d_state int32 [n_rows, W]; d_row int32 [n_envs], or
 * NULL for row i (then n_rows must equal n_envs). n_rows may be smaller or larger than n_envs. An env whose index is
 * negative or >= n_rows, or whose row carries another layout tag, is left untouched (nothing can be reported from the
 * device without a synchronisation). A loaded env gets every field above back; its pool row is clamped into the current
 * parameter pool and its cursor into the trajectory table (a row saved before a smaller locosim_set_param_pool cannot index
 * out of bounds). Its rotation angle is pinned to its episode, so that its reference rows use the saved angle rather than
 * the one drawn for the destination env. The stored observation goes to d_obs fp32 [n_envs, obs_dim] (may be NULL; the
 * rows of envs not loaded are not written). With body or reference outputs registered, d_next_body, the reference keys and
 * d_next_ref of the loaded envs are rewritten as locosim_reset_rows writes them (one more kernel).
 * Not part of a row, and left alone by a load: the diagnostic counters (locosim_get_counters; also the regrouping key,
 * which changes no bit of any result), the caller's applied-force buffers (index them with the same rows), and the
 * handle-wide settings (solver, time limit, parameter pool, registered outputs).
 * A loaded env keeps its own global env id: its next reset draws (traj, sample), the pool row and the rotation angle from
 * the destination's stream at the saved reset counter. Loading a row back into the env it was saved from therefore
 * replays the original bit for bit, auto-resets included, on any launch path; envs forked from one row are identical
 * until their first reset and then diverge.
 * Both calls are stream-ordered, synchronise nothing and allocate nothing: they can be captured in a CUDA graph. d_state
 * must be 16-byte aligned and must not overlap d_obs (or d_row); both are refused. */
#define LS_STATE_VERSION 0x4C530001
#define LS_STATE_TAG 0
#define LS_STATE_EPISODE 2
#define LS_STATE_DR_ROW 3
#define LS_STATE_CURSOR 4
#define LS_STATE_ANGLE 5
#define LS_STATE_EP 8
#define LS_STATE_GOAL 12
#define LS_STATE_QPOS(nv) (16)
#define LS_STATE_QVEL(nv) (16 + (nv))
#define LS_STATE_WARMSTART(nv) (16 + 2 * (nv))
#define LS_STATE_OBS(nv) (16 + 3 * (nv))
#define LS_STATE_WORDS(nv, obs_dim) ((16 + 3 * (nv) + (obs_dim) + 3) / 4 * 4)
int locosim_state_words(const locosim_t* h);
int locosim_save_state(locosim_t* h, const float* d_obs, int32_t* d_state, void* stream);
int locosim_load_state(locosim_t* h, const int32_t* d_state, int n_rows, const int32_t* d_row, float* d_obs, void* stream);

/* Ray casting against every env's geoms, MuJoCo 2.3.7's mj_ray for a batch of rays (what a loco-mujoco user builds
 * rangefinders, height scans, distance-to-obstacle terms and depth or segmentation cameras from). Every env is taken at its
 * stored state (what locosim_get_state returns, the state of info["next_obs"]) with its current parameter-pool row, and the
 * kinematics of the body outputs.
 *   d_pnt, d_vec  fp32 [n_rays, 3] shared by every env, or [n_envs, n_rays, 3] with LS_RAY_PER_ENV: the ray pnt + x vec, in
 *                 the query frame:
 *                   LS_RAY_WORLD    world coordinates (frame_body is not read, but must be a body index)
 *                   LS_RAY_BODY     the frame (xpos, xquat) of body frame_body, as in the body outputs
 *                   LS_RAY_HEADING  at xpos of frame_body, rotated about the world z axis by the yaw of the body's x axis (a
 *                                   heading frame: height scans that turn with the robot but stay level)
 *                   LS_RAY_TRACK    at xpos of frame_body with the world's axes (a tracking camera)
 *   d_dist        fp32 [n_envs, n_rays]: the smallest x >= 0 for which pnt + x vec lies on a selected geom's surface, in units
 *                 of |vec| (a unit vec gives metres), or -1 when nothing is hit, and for a zero vec
 *   d_geom        int32 [n_envs, n_rays]: that geom's index in the compiled model (the ids of the contact list), or -1
 *   d_normal      fp32 [n_envs, n_rays, 3] or NULL: the outward unit normal of the surface at the hit, world frame; zeros when
 *                 nothing is hit. (MuJoCo 2.3.7's mj_ray has no normal: this one is defined here; shading uses it.)
 *   exclude_body  MuJoCo's bodyexclude: the geoms of this body are skipped; -1: none
 *   flags         LS_RAY_STATIC: geoms on bodies welded to the world (no joint on their path to it: MuJoCo's flg_static,
 *                 the floor); LS_RAY_DYNAMIC: every other geom (the robot's); both: every geom
 * Geometry: every geom the engine collides with. Plane, sphere, capsule, ellipsoid, cylinder and box follow MuJoCo 2.3.7's
 * engine_ray.c: a plane is hit from its +z side only, and only within size[0] x size[1] where those are non-zero; a ray that
 * starts inside a solid primitive reports where it leaves it (the smallest non-negative root). A mesh geom is cast against
 * the convex hull of its compiled vertices, the shape the engine collides with (MuJoCo casts against the mesh's own
 * triangles: a non-convex mesh differs in its concave parts); a ray that starts inside a hull reports where it leaves it.
 * Geom groups and rgba are not part of the compiled model, so they select nothing (MuJoCo's geomgroup filter and its
 * skipping of invisible geoms have no counterpart), and visual-only geoms are not there to be hit.
 * A non-finite qpos or qvel of an env gives that env -1 and zeros. NULL d_pnt, d_vec, d_dist or d_geom, n_rays < 1, an
 * unknown frame or flag bit, frame_body or exclude_body out of range, outputs that overlap each other or the inputs, and a
 * launch grid the device cannot take (more than 65535 * 128 rays per env) are refused. The call changes nothing: state, warm
 * start, counters, cursors, random streams, episode statistics and every registered output stay as they were, so a step after
 * it is bit-identical to the same step without it. Stream-ordered, no host synchronisation, no allocation: it can be
 * captured in a CUDA graph (a replay reads the rays and the state as they are then). */
#define LS_RAY_WORLD 0
#define LS_RAY_BODY 1
#define LS_RAY_HEADING 2
#define LS_RAY_TRACK 3
#define LS_RAY_STATIC 1
#define LS_RAY_DYNAMIC 2
#define LS_RAY_PER_ENV 4
int locosim_ray(locosim_t* h, const float* d_pnt, const float* d_vec, int n_rays, int frame, int frame_body,
                int exclude_body, int flags, float* d_dist, int32_t* d_geom, float* d_normal, void* stream);

/* Per-episode goal features (UnitreeA1: cos / sin of the goal direction and the goal speed, GoalDirectionVelocity set in
 * setup() unitreeA1.py:287-291); normally loaded from the reset table, settable for reset(obs=...) (base.py:217-218,633-654).
 * d_goal fp32 [n_envs, 4]. */
int locosim_set_goal(locosim_t* h, const float* d_goal, void* stream);

/* Diagnostics: per-env counters since create: [0]=env steps, [1]=resets, [2]=Newton iterations of the last control
 * step (summed over its sub-steps; also the regrouping key), [3]=contacts of the last sub-step, [4]=terminations caused by
 * a non-finite state, [5..7]=max over control steps of [2] / the last sub-step's contacts / constraint rows.  d_out int32 [n_envs, 8]. */
int locosim_get_counters(locosim_t* h, int32_t* d_out, void* stream);

/* Domain randomisation (replaces DomainRandomizationHandler + per-reset MjModel recompilation,
 * /root/reference/loco_mujoco/utils/domain_randomization.py:191-296, hooked at base.py:183-185): a HOST pool of n_rows
 * parameter sets (row layout: loco_mujoco_b200/domain_randomization.py POOL_FIELDS + meaninertia + 4 user features, row_len
 * floats as float64) is uploaded once; the same mechanism carries multi-model envs (carry tasks: one row per weight,
 * user feature 0 = the weight's mass, observed through LS_OBS_PARAM); every (auto-)reset draws one row per env from the engine's counter-based stream. */
int locosim_param_pool_row_len(const locosim_t* h);
int locosim_set_param_pool(locosim_t* h, const double* pool, int n_rows, int row_len);
/* pool row currently used by each env: d_out int32 [n_envs] */
int locosim_get_param_rows(locosim_t* h, int32_t* d_out, void* stream);

/* Kernels enqueued by one locosim_step: the fused step kernel, preceded (default) by the one-block regrouping kernel that
 * buckets the envs by the solver effort of their previous step (scheduling only; results do not depend on it); one per
 * range of sub-steps with LOCOSIM_RESORT; 1 for the persistent sub-step kernel. */
int locosim_kernels_per_step(const locosim_t* h);

/* Measurement aid (bench.py): non-tensor FP32 FMA throughput of `device` in TFLOP/s, measured with a register-only
 * FMA-chain kernel on all SMs (best of 5). Not part of the simulation path. */
int locosim_measure_fp32_peak(int device, double* tflops_out);

/* Diagnostics of the convex (MPR) narrow phase, process-wide, only counted when the library was created with the environment
 * variable LOCOSIM_DEBUG having bit 8 set: out8[0] = MPR runs, [1] = support calls, [3] = runs that hit the iteration cap. */
int locosim_debug_counters(unsigned long long* out8);

/* Launch geometry chosen for this handle: warps(envs) per block, dynamic shared memory bytes per block, blocks. */
int locosim_launch_info(const locosim_t* h, int* warps_per_block, int* smem_bytes, int* n_blocks);

/* Measurement aid (tools/sm_timeline.py), persistent sub-step kernel only: every later step appends one record of 8 int64 per
 * group to the device buffer d_records [1 + capacity, 8] (d_records[0] counts the records, zero it before the step): SM id,
 * chunk, envs, pop start, group start, group end (%globaltimer, ns), Newton iterations summed over the envs, the largest of
 * them. capacity 0 (or NULL) turns it off. Fails when the handle does not run the persistent kernel. */
int locosim_set_timeline(locosim_t* h, long long* d_records, int capacity);

#ifdef __cplusplus
}
#endif
#endif
