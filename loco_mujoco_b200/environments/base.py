"""
LocoEnv facade over the batched CUDA engine.

Same public surface as the reference's `LocoEnv` (/root/reference/loco_mujoco/environments/base.py:25-969):
`make`, `register`, `get_all_task_names`, `list_registered_loco_mujoco`, `reset`, `step`, `reward`, `is_absorbing`,
`create_dataset`, `play_trajectory`, `load_trajectory`, `get_obs_idx`, `get_all_observation_keys`,
`get_kinematic_obs_mask`, `info.observation_space / action_space`, `dt`; plus the additive kwargs
`num_envs`, `device`, `seed`:

* `num_envs=None` (default): drop-in single-env mode. `reset()` returns a float64 numpy observation, `step(a)` returns
  `(obs, reward, absorbing, info)`; trajectory sampling uses the legacy global numpy RNG exactly like the reference,
  so `np.random.seed(0)` reproduces the reference's golden rollouts (to fp32 tolerance). No auto-reset.
* `num_envs=N`: batched mode. `reset()` -> `obs[N, D]` torch.cuda float32, `step(a[N, nu])` ->
  `(obs, reward, absorbing, info)` with `info["next_obs"]` (the observation to act on after the in-kernel auto-reset).

All physics runs in the CUDA engine (loco_mujoco_b200/csrc); there is no CPU path.
"""
import os
import warnings
from collections import namedtuple
from copy import deepcopy
from itertools import product

import numpy as np

from .. import mjcf, modelpack
from ..engine import DONE_ABSORBING, DONE_TRUNCATED, split_done
from ..task import (TaskSpec, OBS_QPOS, OBS_QVEL, OBS_GOAL, OBS_GRF, OBS_PARAM, GRF_FLOOR, REWARD_NONE, REWARD_TARGET_VELOCITY,
                    REWARD_POS, REWARD_TRACKING)
from ..trajectory import Trajectory
from ..utils.reward import NoReward, CustomReward, TargetVelocityReward, PosReward

# LocoEnv.contacts: torch views of the engine's contact-list buffers (include/locosim.h locosim_set_contact_list_outputs)
ContactList = namedtuple("ContactList", "ncon dist pos frame force geom body dim")


class ObservationType:
    """Subset of mushroom_rl.utils.mujoco.ObservationType used by the in-scope envs."""
    JOINT_POS = "JOINT_POS"
    JOINT_VEL = "JOINT_VEL"
    SITE_ROT = "SITE_ROT"


class Box:
    """Minimal stand-in for mushroom_rl.utils.spaces.Box (low / high / shape)."""

    def __init__(self, low, high):
        self.low = np.array(low, dtype=np.float64)
        self.high = np.array(high, dtype=np.float64)

    @property
    def shape(self):
        return self.low.shape


class MDPInfo:
    def __init__(self, observation_space, action_space, gamma, horizon, dt):
        self.observation_space = observation_space
        self.action_space = action_space
        self.gamma = gamma
        self.horizon = horizon
        self.dt = dt

    @property
    def size(self):
        return self.observation_space.shape + self.action_space.shape

    @property
    def shape(self):
        return self.observation_space.shape + self.action_space.shape


class ObservationHelper:
    """Index bookkeeping of the flat observation (what mushroom's ObservationHelper provides to the reference)."""

    def __init__(self, observation_spec, model):
        self.observation_spec = list(observation_spec)
        self.obs_idx_map = {}
        self.obs_low, self.obs_high = [], []
        self.joint_pos_idx, self.joint_vel_idx = [], []
        i = 0
        for key, name, ot in self.observation_spec:
            n = 9 if ot == ObservationType.SITE_ROT else 1
            self.obs_idx_map[key] = list(range(i, i + n))
            if ot == ObservationType.JOINT_POS:
                j = model.joint_id(name)
                if model.jnt_limited[j]:
                    self.obs_low.append(model.jnt_range[j, 0]); self.obs_high.append(model.jnt_range[j, 1])
                else:
                    self.obs_low.append(-np.inf); self.obs_high.append(np.inf)
                self.joint_pos_idx.append(i)
            else:
                self.obs_low += [-np.inf] * n
                self.obs_high += [np.inf] * n
                if ot == ObservationType.JOINT_VEL:
                    self.joint_vel_idx.append(i)
            i += n
        self.obs_length = i

    def get_all_observation_keys(self):
        return [k for k, _, _ in self.observation_spec]

    def get_from_obs(self, obs, key):
        return obs[self.obs_idx_map[key]]

    def get_joint_pos_from_obs(self, obs):
        return obs[self.joint_pos_idx]

    def get_joint_vel_from_obs(self, obs):
        return obs[self.joint_vel_idx]


def reference_data_root():
    """Directory that holds `environments/data` and `datasets` of a loco_mujoco checkout, or None."""
    if os.environ.get("LOCO_MUJOCO_B200_FORCE_BUNDLED"):
        return None
    cands = [os.environ.get("LOCO_MUJOCO_PATH")]
    try:
        import importlib.util
        spec = importlib.util.find_spec("loco_mujoco")
        if spec is not None and spec.origin:
            cands.append(os.path.dirname(spec.origin))
    except Exception:
        pass
    for c in cands:
        if c and os.path.isdir(os.path.join(c, "environments", "data")):
            return c
    return None


def resolve_time_limit(time_limit, horizon):
    """`time_limit` argument of LocoEnv -> max_episode_steps of the engine (0 = no limit)."""
    if time_limit is None:
        return 0
    if isinstance(time_limit, str):
        if time_limit != "horizon":
            raise ValueError("time_limit must be None, a positive number of control steps or \"horizon\", not %r" % (time_limit,))
        time_limit = horizon
    if isinstance(time_limit, bool) or int(time_limit) != time_limit or time_limit <= 0:
        raise ValueError("time_limit must be a positive number of control steps, not %r" % (time_limit,))
    return int(time_limit)


ASSET_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "assets")


def asset_path(rel):
    """Path of a compiled asset (`<task>.npz`, `dr_pools/<task>.npz`): the package's own ASSET_DIR first, then the
    directories listed in LOCO_MUJOCO_B200_ASSET_PATH (os.pathsep-separated; e.g. the full-body variants shipped as test
    fixtures under tests/golden/full_body). None if no directory has it."""
    extra = [d for d in os.environ.get("LOCO_MUJOCO_B200_ASSET_PATH", "").split(os.pathsep) if d]
    for d in [ASSET_DIR] + extra:
        path = os.path.join(d, rel)
        if os.path.exists(path):
            return path
    return None


class LocoEnv:
    """Base class of all batched locomotion environments."""

    _registered_envs = dict()
    _terrain_supported = False      # (the robots whose compiled models may carry a terrain: UnitreeA1)

    def __init__(self, xml_handles, action_spec, observation_spec, collision_groups=None, gamma=0.99, horizon=1000,
                 n_substeps=10, reward_type=None, reward_params=None, traj_params=None, random_start=True,
                 init_step_no=None, timestep=0.001, use_foot_forces=False, default_camera_mode="follow",
                 use_absorbing_states=True, domain_randomization_config=None, parallel_dom_rand=True,
                 N_worker_per_xml_dom_rand=4, num_envs=None, device="cuda:0", seed=0, env_id_offset=0,
                 compiled_model=None, copy_outputs=True, convex_collisions=True, warps_per_block=None, time_limit=None,
                 truncate_at_trajectory_end=False, terrain=None, **viewer_params):
        if type(xml_handles) != list:
            xml_handles = [xml_handles]
        self._xml_handles = xml_handles
        # several handles = a multi-model env (carry tasks: one model per weight; base.py:86-88,183-191). All models share
        # topology and sizes, so the engine runs them as rows of the parameter pool (one row per model).
        # use_foot_forces (base.py:93-98 of the reference): n_intermediate_steps x mj_step(1) with a contact-force hook
        # after each one. The engine always runs n_substeps physics steps per control step; dt is unchanged.
        self._collision_groups = list(collision_groups) if collision_groups else []
        self._domain_rand_config = domain_randomization_config
        self._domain_rand_pool_size = viewer_params.pop("domain_randomization_pool_size", 64)
        # render(): the reference's viewer settings that a headless frame uses (camera_params["follow"], width, height)
        self._camera_params = dict(viewer_params.get("camera_params") or {})
        self._render_size = (int(viewer_params.get("width", 640)), int(viewer_params.get("height", 480)))
        self._domain_rand = None
        self._timestep = timestep
        self._n_substeps = n_substeps
        self._n_intermediate_steps = 1
        self._use_foot_forces = use_foot_forces
        if compiled_model is not None:
            self._models = list(compiled_model) if isinstance(compiled_model, (list, tuple)) else [compiled_model]
        else:
            self._models = [mjcf.compile_model(h, timestep=timestep) for h in xml_handles]
        # terrain: a height field (loco_mujoco_b200.terrain.HeightField) attached to the compiled model as its last geom
        # (include/locosim.h locosim_set_terrain_origin); UnitreeA1 only
        if terrain is not None:
            if domain_randomization_config is not None:
                # (the randomised parameter pools are built from models without the terrain geom: their rows would not
                # match the terrain model's)
                raise NotImplementedError("terrain together with domain_randomization_config is not supported")
            if not self._terrain_supported:
                raise NotImplementedError("terrain is implemented for UnitreeA1 only (its floor-colliding geoms are "
                                          "spheres, capsules, cylinders and boxes), not for %s" % type(self).__name__)
            from .. import terrain as _terrain
            self._models = [_terrain.attach(m, terrain) for m in self._models]
        self._terrain_origin = None
        self._model = self._models[0]
        if timestep is None:
            self._timestep = self._model.opt_timestep
        self._model_user_features = [()] * len(self._models)     # per model: values observable through OBS_PARAM
        if len(self._models) > 1 and domain_randomization_config is not None:
            raise NotImplementedError("domain randomisation of a multi-model env")
        self._action_spec = list(action_spec) if len(action_spec) else list(self._model.actuator_names)
        self._action_indices = [self._model.actuator_id(n) for n in self._action_spec]
        if sorted(self._action_indices) != list(range(self._model.nu)):
            raise NotImplementedError("action_spec must cover all actuators of the (modified) model")
        self.obs_helper = ObservationHelper(observation_spec, self._model)
        self.obs_helpers = [self.obs_helper]
        lo = self._model.actuator_ctrlrange[self._action_indices, 0].copy()
        hi = self._model.actuator_ctrlrange[self._action_indices, 1].copy()
        self.info = MDPInfo(Box(self.obs_helper.obs_low, self.obs_helper.obs_high), Box(lo, hi), gamma, horizon, self.dt)

        self._reward_type, self._reward_params = reward_type, reward_params
        self._reward_function = self._get_reward_function(reward_type, reward_params)
        self.info.observation_space = Box(*self._get_observation_space())
        low, high = self.info.action_space.low.copy(), self.info.action_space.high.copy()
        self.norm_act_mean = (high + low) / 2.0
        self.norm_act_delta = (high - low) / 2.0
        self.info.action_space.low[:] = -1.0
        self.info.action_space.high[:] = 1.0

        self._dataset = None
        self.trajectories = None
        if traj_params:
            self.load_trajectory(traj_params)
        self._random_start = random_start
        self._init_step_no = init_step_no
        self._use_absorbing_states = use_absorbing_states

        self._num_envs = num_envs
        self._device = device
        self._seed = seed
        self._env_id_offset = env_id_offset
        # Batched mode: the engine writes every step into the same device buffers. copy_outputs=True (default) hands the
        # caller private copies (two device-to-device copies per step), so that appending them to a rollout buffer is safe;
        # copy_outputs=False returns views that are only valid until the next step()/reset() (zero-copy, benchmark use).
        self._copy_outputs = bool(copy_outputs)
        # convex_collisions=False drops the mesh-mesh / box-mesh candidate pairs (bone against bone: mjc_Convex / MPR) from the
        # engine's pair table: faster (HumanoidTorque: ~3x), but not what the reference simulates. Default: on.
        self._convex_collisions = bool(convex_collisions)
        # launch geometry of the step kernel (envs per block); None = the engine's choice. Scheduling only (MixedBatch uses it)
        self._warps_per_block = warps_per_block
        # Time limit (include/locosim.h locosim_set_time_limit), off by default like in the reference, whose env never
        # truncates (there the consumer enforces `horizon`): time_limit = None, a number of control steps, or "horizon" (= the
        # `horizon` argument); truncate_at_trajectory_end ends an episode where its mocap trajectory does. With either on,
        # step() reports `info["truncated"]`, and batched envs reset truncated episodes in the same step like fallen ones.
        self._max_episode_steps = resolve_time_limit(time_limit, horizon)
        self._truncate_at_trajectory_end = bool(truncate_at_trajectory_end)
        # applied forces (xfrc_applied / qfrc_applied below): allocated and registered with the engine on first access
        self._xfrc_applied = None
        self._qfrc_applied = None
        # body outputs (body_state / next_body_state below): allocated and registered with the engine on first access
        self._body_state = None
        self._next_body_state = None
        # contact outputs (contact_wrench below): allocated and registered with the engine on first access
        self._contact_wrench = None
        # dof outputs (dof_outputs below): allocated and registered with the engine on first access
        self._dof_outputs = None
        # contact list (contacts below): (ncon, con, con_id) allocated and registered with the engine on first access
        self._contact_list = None
        # reference outputs (reference_body_state / next_reference_body_state below): likewise
        self._reference_body_state = None
        self._next_reference_body_state = None
        self._engine = None
        self._obs = None

    @property
    def time_limited(self):
        return self._max_episode_steps > 0 or self._truncate_at_trajectory_end

    # ---------------------------------------------------------------------------------------------------
    # construction helpers
    # ---------------------------------------------------------------------------------------------------
    @property
    def dt(self):
        return self._timestep * self._n_intermediate_steps * self._n_substeps

    @property
    def num_envs(self):
        return 1 if self._num_envs is None else self._num_envs

    @property
    def batched(self):
        return self._num_envs is not None

    def load_trajectory(self, traj_params, warn=True):
        if self.trajectories is not None:
            warnings.warn("New trajectories loaded, which overrides the old ones.", RuntimeWarning)
        if "processed" in traj_params:
            self.trajectories = _ProcessedTrajectory(traj_params["processed"])
        else:
            self.trajectories = Trajectory(keys=self.get_all_observation_keys(),
                                           low=self.info.observation_space.low,
                                           high=self.info.observation_space.high,
                                           joint_pos_idx=self.obs_helper.joint_pos_idx,
                                           interpolate_map=self._interpolate_map,
                                           interpolate_remap=self._interpolate_remap,
                                           interpolate_map_params=self._get_interpolate_map_params(),
                                           interpolate_remap_params=self._get_interpolate_remap_params(),
                                           warn=warn, **traj_params)
        self._engine = None

    def get_all_observation_keys(self):
        return self.obs_helper.get_all_observation_keys()

    # ---------------------------------------------------------------------------------------------------
    # TaskSpec: flatten obs / done / reward / reset table for the engine
    # ---------------------------------------------------------------------------------------------------
    def _has_fallen_terms(self):
        """list of (observation key, low, high): fallen if value < low or value > high."""
        raise NotImplementedError

    def _goal_features(self, sample):
        """Per-episode constant observation features derived from a trajectory sample (goal-conditioned envs)."""
        return []

    def _n_goal(self):
        return 0

    def _obs_sources(self):
        """(src_type, src_idx) for every entry of the final observation vector."""
        types, idxs = [], []
        for key, name, ot in self.obs_helper.observation_spec[2:]:
            if ot == ObservationType.JOINT_POS:
                types.append(OBS_QPOS); idxs.append(self._model.joint_id(name))
            elif ot == ObservationType.JOINT_VEL:
                types.append(OBS_QVEL); idxs.append(self._model.joint_id(name))
            else:
                raise NotImplementedError(ot)
        return types, idxs

    def _reward_spec(self):
        rt = self._reward_type
        if rt is None:
            return REWARD_NONE, [], []
        if rt == "target_velocity":
            return REWARD_TARGET_VELOCITY, [self.get_obs_idx("dq_pelvis_tx")[0]], [self._reward_params["target_velocity"]]
        if rt == "x_pos":
            return REWARD_POS, [self.get_obs_idx("q_pelvis_tx")[0]], []
        if rt == "custom":
            return REWARD_NONE, [], []      # evaluated on the host from the returned tensors
        if rt == "tracking":
            return REWARD_TRACKING, [], []  # weights travel in TaskSpec.tracking
        raise NotImplementedError(rt)

    def _reset_table(self):
        """[n_traj, T, nq + nv + n_goal] from the (interpolated) trajectories."""
        tr = self.trajectories
        nq = self._model.nq
        n_traj, T = tr.number_of_trajectories, tr.trajectory_length
        table = np.zeros((n_traj, T, 2 * nq + self._n_goal()))
        spec = self.obs_helper.observation_spec
        for k, (key, name, ot) in enumerate(spec):
            arr = tr.trajectories[tr.keys.index(key)]
            if ot == ObservationType.JOINT_POS:
                table[:, :, self._model.joint_id(name)] = arr
            elif ot == ObservationType.JOINT_VEL:
                table[:, :, nq + self._model.joint_id(name)] = arr
        if self._n_goal():
            for i in range(n_traj):
                for j in range(T):
                    sample = [obs[i][j] for obs in tr.trajectories]
                    table[i, j, 2 * nq:] = self._goal_features(sample)
        return table

    def task_spec(self):
        types, idxs = self._obs_sources()
        keys_to_idx = {}
        done_terms = []
        for key, lo, hi in self._has_fallen_terms():
            done_terms.append((self.get_obs_idx(key)[0], lo, hi))
        rtype, rints, rparams = self._reward_spec()
        spec = self.obs_helper.observation_spec
        recenter = [self._model.joint_id(spec[0][1]), self._model.joint_id(spec[1][1])]
        if self.trajectories is None:
            raise ValueError("the CUDA engine needs trajectory data for resets (pass traj_params)")
        n_grf, grf_group = self._grf_spec()
        types = list(types) + [OBS_GRF] * (3 * n_grf)           # mean ground forces, then per-model features (weight)
        idxs = list(idxs) + list(range(3 * n_grf))
        n_user = len(self._model_user_features[0])
        types += [OBS_PARAM] * n_user
        idxs += list(range(n_user))
        return TaskSpec(types, idxs, done_terms, rtype, rints, rparams, self.norm_act_mean, self.norm_act_delta,
                        self._n_substeps, self._reset_table(), self._n_goal(), recenter, self._use_absorbing_states,
                        act_idx=self._action_indices, n_grf=n_grf, grf_group=grf_group, random_rot=self._random_rot_spec(),
                        tracking=self._tracking_params())

    TRACKING_DEFAULTS = dict(w_pose=0.7, k_pose=2.0, w_vel=0.3, k_vel=0.1)

    def _tracking_params(self):
        """(w_pose, k_pose, w_vel, k_vel) of reward_type="tracking" (this package's mocap-tracking reward, see
        include/locosim_task.h LS_REWARD_TRACKING; the reference has no reward that reads the trajectory)."""
        if self._reward_type != "tracking":
            return None
        prm = dict(self.TRACKING_DEFAULTS, **(self._reward_params or {}))
        return [prm["w_pose"], prm["k_pose"], prm["w_vel"], prm["k_vel"]]

    def _random_rot_spec(self):
        """None, or (qpos index of the yaw joint, dof indices of the root x / y velocity): setup_random_rot."""
        return None

    def domain_randomization_pool(self):
        """[K, P] parameter pool: K consecutive randomised recompilations of the model (see domain_randomization.py)."""
        if self._domain_rand is None:
            from ..domain_randomization import DomainRandomizationHandler
            if self._xml_handles[0] is None:
                self._dr_pool = self._bundled_dr_pool()
                self._domain_rand = "bundled"
                return self._dr_pool
            self._domain_rand = DomainRandomizationHandler([self._xml_handles[0].copy()], self._domain_rand_config,
                                                           timestep=self._timestep)
            self._dr_pool = self._domain_rand.build_pool(self._domain_rand_pool_size)
        return self._dr_pool

    def _bundled_dr_pool(self):
        """Without the MJCF sources (bundled assets only, e.g. on the GPU box) the randomised recompilations cannot be
        made; for the reference's shipped YAML configs a pre-built seeded pool is bundled (tools/build_dr_pools.py)."""
        import json
        task_id = getattr(self, "_task_id", None)
        path = asset_path(os.path.join("dr_pools", "%s.npz" % task_id)) if task_id is not None else None
        if path is None:
            raise ValueError("domain randomisation needs the MJCF source (a loco_mujoco checkout); no pre-built pool is "
                             "bundled for %s" % task_id)
        d = np.load(path, allow_pickle=False)
        meta = json.loads(str(d["meta"]))
        conf = self._domain_rand_config
        ok = (isinstance(conf, str) and os.path.basename(conf) == meta["yaml"]) or conf == meta["config_used"] or \
            conf == meta["config_shipped"]
        if not ok:
            raise ValueError("the bundled pool of %s was built for %s; other configs need the MJCF source"
                             % (task_id, meta["yaml"]))
        return np.asarray(d["pool"], dtype=np.float64)

    def model_pool(self):
        """[n_models, P] parameter pool of a multi-model env (one row per model incl. its user features)."""
        from ..domain_randomization import pool_row
        return np.stack([pool_row(m, u) for m, u in zip(self._models, self._model_user_features)])

    def _get_engine(self):
        if self._engine is None:
            from ..engine import CudaEngine
            import torch
            dev = torch.device(self._device)
            self._engine = CudaEngine(modelpack.pack(self._model, convex_pairs=self._convex_collisions),
                                      self.task_spec().pack(), self.num_envs,
                                      device=dev.index or 0, seed=self._seed, env_id_offset=self._env_id_offset,
                                      warps_per_block=self._warps_per_block)
            if self._domain_rand_config is not None:
                self._engine.set_param_pool(self.domain_randomization_pool())
            elif len(self._models) > 1 or len(self._model_user_features[0]):
                self._engine.set_param_pool(self.model_pool())
            if self.time_limited:
                self._engine.set_time_limit(self._max_episode_steps, self._truncate_at_trajectory_end)
            if self._xfrc_applied is not None or self._qfrc_applied is not None:
                self._engine.set_applied_forces(self._xfrc_applied, self._qfrc_applied)
            if self._terrain_origin is not None:
                self._engine.set_terrain_origin(self._terrain_origin)
            if self._body_state is not None:
                self._engine.set_body_outputs(self._body_state, self._next_body_state)
            if self._contact_wrench is not None:
                self._engine.set_contact_outputs(self._contact_wrench)
            if self._dof_outputs is not None:
                self._engine.set_dof_outputs(self._dof_outputs)
            if self._contact_list is not None:
                self._engine.set_contact_list_outputs(*self._contact_list[:3])
            if self._reference_body_state is not None:
                self._engine.set_reference_outputs(self._reference_body_state, self._next_reference_body_state)
        return self._engine

    # ---------------------------------------------------------------------------------------------------
    # applied forces (MuJoCo's mjData.xfrc_applied / qfrc_applied, include/locosim.h locosim_set_applied_forces)
    # ---------------------------------------------------------------------------------------------------
    def body_index(self, name):
        """Row of body `name` in `xfrc_applied`, `body_state`, `next_body_state` and `contact_wrench` (an index of the compiled
        model).
        ValueError for an unknown name and for a body that fuse_static merged into its parent; the message then names the
        parent."""
        return self._model.body_index(name)

    @property
    def xfrc_applied(self):
        """float32 torch tensor [num_envs, nbody, 6] on the env's device: per body a force (3) then a torque (3) in world
        coordinates, applied at the body's centre of mass in every dynamics evaluation of every later step (row 0, the world,
        is ignored). Write into it in place (also between replays of a captured CUDA graph); it keeps its values until you
        change them, except that every reset of an env (reset(), the auto-reset of a fallen or truncated env) zeroes that
        env's rows. Allocated zeroed and registered with the engine on first access: an env that never touches it runs the
        step without applied forces."""
        if self._xfrc_applied is None:
            self._xfrc_applied = self._new_applied((self.num_envs, self._model.nbody, 6))
        return self._xfrc_applied

    @property
    def qfrc_applied(self):
        """float32 torch tensor [num_envs, nq] of generalised forces added to the joint forces in every dynamics
        evaluation (MuJoCo's qfrc_applied). Same life cycle as `xfrc_applied`."""
        if self._qfrc_applied is None:
            self._qfrc_applied = self._new_applied((self.num_envs, self._model.nv))
        return self._qfrc_applied

    @property
    def terrain(self):
        """The height field of this env (loco_mujoco_b200.terrain.HeightField), or None."""
        return getattr(self._model, "hfield", None)

    @property
    def terrain_origin(self):
        """float32 torch tensor [num_envs, 2] on the env's device: per env the terrain point (x, y) that lies under the env's
        world origin (its reset spot); env i sees the height field translated by -terrain_origin[i]. Write into it in place
        (also between replays of a captured CUDA graph); every later step and query reads it. Resets do not change it: root
        x / y restart at 0, so an env restarts on the same terrain point. Allocated zeroed and registered with the engine on
        first access (touch it before capturing a step in a CUDA graph). Only for an env made with `terrain=`."""
        if self.terrain is None:
            raise ValueError("this env has no terrain (LocoEnv.make(..., terrain=HeightField))")
        if self._terrain_origin is None:
            import torch
            eng = self._get_engine()
            t = torch.zeros((self.num_envs, 2), dtype=torch.float32, device=eng.device)
            eng.set_terrain_origin(t)
            self._terrain_origin = t
        return self._terrain_origin

    def _new_applied(self, shape):
        import torch
        eng = self._get_engine()
        t = torch.zeros(shape, dtype=torch.float32, device=eng.device)
        x, q = (t, self._qfrc_applied) if len(shape) == 3 else (self._xfrc_applied, t)
        eng.set_applied_forces(x, q)
        return t

    # ---------------------------------------------------------------------------------------------------
    # body outputs (MuJoCo's xpos / xquat / mj_objectVelocity, include/locosim.h locosim_set_body_outputs)
    # ---------------------------------------------------------------------------------------------------
    @property
    def body_state(self):
        """float32 torch tensor [num_envs, nbody, BODY_DIM = 13] on the env's device, rewritten by every step: per body (row
        `body_index(name)`) the world position of the body frame (3), its orientation quaternion w, x, y, z (4), its angular
        velocity (3) and the linear velocity of the body-frame origin (3), both in world coordinates (mj_objectVelocity with
        mjOBJ_XBODY: the frame origin, not the centre of mass). It describes the state the step's observation describes: for
        an env that ended, its terminal state; for an env whose state became non-finite, zeros. Values are those of an
        mj_forward on that state (MuJoCo's mjData after mj_step still holds the start of the last sub-step). Allocated and
        registered, together with `next_body_state`, on first access of either: an env that never touches them computes
        nothing extra. Touch them before capturing a step in a CUDA graph: a graph captured before the first access does
        not write them (capture it again afterwards)."""
        if self._body_state is None:
            self._new_body_outputs()
        return self._body_state

    @property
    def next_body_state(self):
        """Like `body_state`, for the state the env acts from next: after a step's auto-reset (rows of envs that did not
        reset equal `body_state`), after reset() and after reset(obs=...)."""
        if self._next_body_state is None:
            self._new_body_outputs()
        return self._next_body_state

    def _new_body_outputs(self):
        import torch
        from ..engine import BODY_DIM
        eng = self._get_engine()
        shape = (self.num_envs, self._model.nbody, BODY_DIM)
        self._body_state = torch.zeros(shape, dtype=torch.float32, device=eng.device)
        self._next_body_state = torch.zeros(shape, dtype=torch.float32, device=eng.device)
        eng.set_body_outputs(self._body_state, self._next_body_state)

    # ---------------------------------------------------------------------------------------------------
    # contact outputs (MuJoCo's mj_contactForce summed per body, include/locosim.h locosim_set_contact_outputs)
    # ---------------------------------------------------------------------------------------------------
    @property
    def contact_wrench(self):
        """float32 torch tensor [num_envs, nbody, CONTACT_DIM = 6] on the env's device, rewritten by every step: per body (row
        `body_index(name)`) the force (3) and the torque (3) that all of the body's contacts exert on it, in world
        coordinates, the torque about the body-frame origin xpos (the point of `body_state`'s linear velocity; not the centre
        of mass, and not the subtree_com convention of MuJoCo's cfrc_ext). Each contact's force is mj_contactForce's (every
        component of its condim, torsional and rolling included), turned into the world frame; it acts with + on geom2's
        body and with - on geom1's, so a self contact appears in two rows with opposite signs. Row 0 (the world) is zero.
        The values are the MEAN over the step's sub-steps (each sub-step's last dynamics evaluation, the window of the
        foot-force observation), not MuJoCo's last sub-step; contacts past the engine's per-env cap are not in the sum. It
        describes the step that produced the observation: for an env that ended, its terminal step; for an env whose state
        became non-finite, zeros. reset() does not write it. Allocated zeroed and registered on first access: an env that
        never touches it computes nothing extra. A step captured in a CUDA graph before the first access writes it from
        the next replay on."""
        if self._contact_wrench is None:
            import torch
            from ..engine import CONTACT_DIM
            eng = self._get_engine()
            t = torch.zeros((self.num_envs, self._model.nbody, CONTACT_DIM), dtype=torch.float32, device=eng.device)
            eng.set_contact_outputs(t)
            self._contact_wrench = t
        return self._contact_wrench

    # ---------------------------------------------------------------------------------------------------
    # dof outputs (MuJoCo's qfrc_actuator / qfrc_constraint / qacc, include/locosim.h locosim_set_dof_outputs)
    # ---------------------------------------------------------------------------------------------------
    @property
    def dof_outputs(self):
        """float32 torch tensor [num_envs, nq, DOF_DIM = 3] on the env's device, rewritten by every step: per dof (the qvel
        layout of the state; every model here has nq == nv) MuJoCo's qfrc_actuator (the actuators' gear * force, ctrlrange
        and forcerange clamps applied), qfrc_constraint (J^T of the constraint forces: contacts, joint limits, friction
        loss) and qacc (the constrained acceleration; for the Euler integrator not the implicit-damping solve it advances
        with). The values are the MEAN over the step's sub-steps (each sub-step's last dynamics evaluation), not MuJoCo's
        last sub-step. It describes the step that produced the observation: for an env that ended, its terminal step; for
        an env whose state became non-finite, zeros. reset() does not write it. Allocated zeroed and registered on first
        access: an env that never touches it computes nothing extra. A step captured in a CUDA graph before the first
        access writes it from the next replay on."""
        if self._dof_outputs is None:
            import torch
            from ..engine import DOF_DIM
            eng = self._get_engine()
            t = torch.zeros((self.num_envs, self._model.nq, DOF_DIM), dtype=torch.float32, device=eng.device)
            eng.set_dof_outputs(t)
            self._dof_outputs = t
        return self._dof_outputs

    # ---------------------------------------------------------------------------------------------------
    # contact list (MuJoCo's d.contact and mj_contactForce, include/locosim.h locosim_set_contact_list_outputs)
    # ---------------------------------------------------------------------------------------------------
    @property
    def contacts(self):
        """The contact list of each env, rewritten by every step: a ContactList of torch views on the env's device, C =
        the engine's per-env contact cap (16):
            ncon   int32 [num_envs]           contacts in the list
            dist   float32 [num_envs, C]      signed distance (negative: penetration)
            pos    float32 [num_envs, C, 3]   contact position, world frame
            frame  float32 [num_envs, C, 3, 3] rows n, t1, t2 of the contact frame (n points from geom1 to geom2)
            force  float32 [num_envs, C, 6]   mj_contactForce's contact-frame force (normal, tangents, torsion, rolling;
                                              zeros past dim); it acts on geom2, its negative on geom1
            geom   int32 [num_envs, C, 2]     geom1, geom2: indices of the compiled model (`geom_index`, `geom_names`)
            body   int32 [num_envs, C, 2]     their bodies (`body_index`, the rows of `contact_wrench` and `body_state`)
            dim    int32 [num_envs, C]        condim of the contact
        The list is the one MuJoCo's mjData holds after mj_step, the contacts and forces of the step's LAST sub-step (its
        last dynamics evaluation), in the engine's list order (the compiled pair table's, as MuJoCo's); `contact_wrench` is
        instead the mean over all sub-steps, summed per body. Contacts past the cap are dropped: ncon == C is the only sign.
        Rows at and past ncon hold zeros and ids of -1. It describes the step that produced the observation: for an env
        that ended, its terminal step; for an env whose state became non-finite, ncon = 0. reset(), set_state() and
        load_state() do not write it. Allocated and registered on first access: an env that never touches it computes
        nothing extra. A step captured in a CUDA graph before the first access writes it from the next replay on."""
        if self._contact_list is None:
            import torch
            from ..engine import CONLIST_DIM, CONLIST_ID_DIM, CONLIST_COLUMNS as F, CONLIST_ID_COLUMNS as I
            eng = self._get_engine()
            n, C, dev = self.num_envs, eng.max_contacts, eng.device
            ncon = torch.zeros((n,), dtype=torch.int32, device=dev)
            con = torch.zeros((n, C, CONLIST_DIM), dtype=torch.float32, device=dev)
            con_id = torch.full((n, C, CONLIST_ID_DIM), -1, dtype=torch.int32, device=dev)
            eng.set_contact_list_outputs(ncon, con, con_id)
            col = lambda t, c: t[:, :, c[0]:c[0] + c[1]]      # noqa: E731
            self._contact_list = (ncon, con, con_id, ContactList(
                ncon=ncon, dist=con[:, :, F["dist"][0]], pos=col(con, F["pos"]),
                frame=col(con, F["frame"]).unflatten(-1, (3, 3)), force=col(con, F["force"]), geom=col(con_id, I["geom"]),
                body=col(con_id, I["body"]), dim=con_id[:, :, I["dim"][0]]))
        return self._contact_list[3]

    @property
    def geom_names(self):
        """Names of the compiled model's geoms, by index (the ids of `contacts.geom`; None for an unnamed geom). Geoms that
        take part in no collision (contype and conaffinity 0: visual only) are dropped by the compiler and are not there."""
        return list(self._model.geom_names)

    def geom_index(self, name):
        """Index of geom `name` in the compiled model (as `contacts.geom` holds it). ValueError for an unknown name and for a
        visual-only geom, which the compiler drops."""
        if name is not None and name in self._model.geom_names:
            return self._model.geom_names.index(name)
        raise ValueError("unknown geom %r (visual-only geoms, contype = conaffinity = 0, are not compiled; geoms of the "
                         "compiled model: %s)" % (name, ", ".join(str(g) for g in self._model.geom_names)))

    # ---------------------------------------------------------------------------------------------------
    # reference outputs (the mocap clip's body outputs, include/locosim.h locosim_set_reference_outputs)
    # ---------------------------------------------------------------------------------------------------
    @property
    def reference_body_state(self):
        """float32 torch tensor [num_envs, nbody, BODY_DIM = 13] on the env's device, rewritten by every step: the expert's
        body state at each env's point in its mocap clip, in the layout and rows of `body_state`. A row is the `body_state`
        row of the state that a reset onto the trajectory sample at the env's cursor would give: root x / y zeroed, the
        rotation of the env's episode (setup_random_rot), the env's parameter-pool row. Right after a reset it equals
        `next_body_state` bit for bit. Positions are root-x/y-relative: subtract the simulated root's x / y before comparing,
        e.g. for foot row f and root row r
            sim = body_state[:, f, :3].clone(); sim[:, :2] -= body_state[:, r, :2]
            err = (sim - reference_body_state[:, f, :3]).norm(dim=-1)
        It describes the state the step's observation describes: for an env that ended, the sample its terminal step
        reached; zeros for an env whose state became non-finite. The cursor advances one sample per step only under
        reward_type="tracking" or truncate_at_trajectory_end=True; with neither the reference would stay on the reset sample,
        so this raises ValueError. Allocated and registered, together with `next_reference_body_state`, on first access of
        either. Touch them before capturing a step in a CUDA graph (capture it again afterwards otherwise)."""
        if self._reference_body_state is None:
            self._new_reference_outputs()
        return self._reference_body_state

    @property
    def next_reference_body_state(self):
        """Like `reference_body_state`, for the state the env acts from next: after a step's auto-reset (rows of envs that
        did not reset equal `reference_body_state`) and after reset(). reset(obs=...) moves no cursor and leaves it alone."""
        if self._next_reference_body_state is None:
            self._new_reference_outputs()
        return self._next_reference_body_state

    def _check_reference_phase(self):
        if self._reward_type != "tracking" and not self._truncate_at_trajectory_end:
            raise ValueError("the reference outputs follow the trajectory cursor, which advances only under "
                             "reward_type=\"tracking\" or truncate_at_trajectory_end=True: make the env with one of them")

    def _new_reference_outputs(self):
        import torch
        from ..engine import BODY_DIM
        self._check_reference_phase()
        eng = self._get_engine()
        shape = (self.num_envs, self._model.nbody, BODY_DIM)
        ref = torch.zeros(shape, dtype=torch.float32, device=eng.device)
        nxt = torch.zeros(shape, dtype=torch.float32, device=eng.device)
        eng.set_reference_outputs(ref, nxt)
        self._reference_body_state, self._next_reference_body_state = ref, nxt

    def create_dataset_bodies(self):
        """The expert side of a body-space discriminator, built on the device: dict of float32 torch tensors body_states /
        next_body_states [n, nbody, BODY_DIM], row-aligned with `create_dataset_device()` (states / next_states / last): row
        r holds the body state of the reset onto dataset row r's trajectory sample, and of the next sample. Rotation angle
        0, the compiled model's own parameters; positions root-x/y-relative as in `reference_body_state`."""
        body, nxt = self._get_engine().create_dataset_bodies()
        return dict(body_states=body, next_body_states=nxt)

    # ---------------------------------------------------------------------------------------------------
    # inverse dynamics (MuJoCo's mj_inverse, include/locosim.h locosim_inverse)
    # ---------------------------------------------------------------------------------------------------
    def dof_index(self, joint_name):
        """Column of joint `joint_name`'s dof in `qfrc_applied`, `dof_outputs`, `inverse_dynamics()` and
        `create_dataset_inverse()` (every model here has one dof per joint, in the qvel order of the state). ValueError for
        an unknown name."""
        names = list(self._model.jnt_names)
        if joint_name not in names:
            raise ValueError("no joint %r in the model (joints: %s)" % (joint_name, ", ".join(names)))
        return names.index(joint_name)

    def inverse_dynamics(self, qacc):
        """MuJoCo's mj_inverse (2.3.7, continuous time) of every env at its current state, the state of info["next_obs"]
        (the one the env acts from next), with its parameter-pool row: float32 torch tensor [num_envs, nq] on the env's
        device,
            qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint(qacc)
        where qfrc_constraint is J^T of the soft-constraint forces that `qacc` implies at the state (contacts, joint limits,
        friction loss). Actuator forces, `qfrc_applied` and `xfrc_applied` are not subtracted, so at the engine's own
        forward solution it is the actuator force plus the applied forces (the root dofs' entries: the "hand of god" force
        a motion needs). `qacc`: float32 [num_envs, nq] on the env's device, in the qvel layout (`dof_index`). A non-finite
        state or qacc gives that env a row of zeros. Changes nothing in the env."""
        import torch
        eng = self._get_engine()
        if not isinstance(qacc, torch.Tensor):
            raise ValueError("qacc must be a float32 torch tensor [num_envs, nq] on %s" % eng.device)
        return eng.inverse(qacc)

    def create_dataset_inverse(self):
        """The joint-space forces the mocap clip needs, built on the device: float32 torch tensor [n, nq], row-aligned with
        `create_dataset_device()` and `create_dataset_bodies()`. Row r is `inverse_dynamics` at the reset state of dataset
        row r's trajectory sample (rotation angle 0, the compiled model's own parameters) at the forward-difference
        acceleration to the next sample, qacc = (qvel[next] - qvel) * float32(1 / (timestep * n_substeps)). Columns of
        actuated joints hold the torque the clip requires; those of the unactuated root dofs, the residual force that
        measures how physically consistent the clip is on this robot."""
        return self._get_engine().create_dataset_inverse()

    # ---------------------------------------------------------------------------------------------------
    # dynamics terms (MuJoCo's qM / qfrc_bias / qfrc_passive / subtree_com / mj_jacBody, include/locosim.h
    # locosim_dynamics_terms)
    # ---------------------------------------------------------------------------------------------------
    DYNAMICS_TERMS = ("mass_matrix", "bias", "passive", "com", "body_jacobian", "com_jacobian")

    def dynamics_terms(self, mass_matrix=True, bias=True, passive=True, com=True, body_jacobian=False, com_jacobian=False,
                       out=None):
        """The model-based terms of every env at its current state, the state of info["next_obs"], with its parameter-pool
        row (MuJoCo 2.3.7's meaning), as a dict of float32 torch tensors on the env's device, one key per term asked for:
            mass_matrix    [num_envs, nq, nq]        M(q) of mj_fullM, dof_armature on the diagonal
            bias           [num_envs, nq]            qfrc_bias = C(q, qvel) qvel + g(q) (mj_rne at qacc = 0)
            passive        [num_envs, nq]            qfrc_passive = -stiffness (q - q_spring) - damping qvel
            com            [num_envs, 4]             the whole-robot centre of mass (x, y, z) and the total mass, a carried
                                                     weight included (both follow the env's pool row)
            body_jacobian  [num_envs, nbody, 6, nq]  mj_jacBody at each body's origin xpos (not its CoM), world frame:
                                                     rows 0-2 angular, rows 3-5 linear, so body_jacobian @ qvel gives
                                                     body_state[..., 7:13]; body 0 (the world) is zeros
            com_jacobian   [num_envs, 3, nq]         d(com) / dq (mj_jacSubtreeCom of the robot)
        so that, away from contacts and joint limits, M qacc + bias - passive = inverse_dynamics(qacc). Dof axes are in the
        qvel layout (`dof_index(joint)`), body axes in the model's body order (`body_index(name)`). A non-finite state gives
        that env zero rows. `out`: the dict of an earlier call, filled in place and returned (a graph-captured loop then
        allocates nothing); terms it lacks are allocated. Changes nothing in the env."""
        eng = self._get_engine()
        n, nq = self.num_envs, self._model.nq
        shapes = dict(mass_matrix=(n, nq, nq), bias=(n, nq), passive=(n, nq), com=(n, 4),
                      body_jacobian=(n, self._model.nbody, 6, nq), com_jacobian=(n, 3, nq))
        want = dict(mass_matrix=mass_matrix, bias=bias, passive=passive, com=com, body_jacobian=body_jacobian,
                    com_jacobian=com_jacobian)
        out, got = self._query_outputs("dynamics_terms", self.DYNAMICS_TERMS, out, want, shapes, eng.device)
        eng.dynamics_terms(M=got["mass_matrix"], bias=got["bias"], passive=got["passive"], com=got["com"],
                           jac=got["body_jacobian"], jac_com=got["com_jacobian"])
        return out

    # ---------------------------------------------------------------------------------------------------
    # forward dynamics under an action (MuJoCo's mj_forward + mj_rnePostConstraint: qacc, cacc, cfrc_int, cfrc_ext,
    # include/locosim.h locosim_forward)
    # ---------------------------------------------------------------------------------------------------
    FORWARD_OUTPUTS = ("dof", "body_acc", "cfrc_int", "cfrc_ext")

    def forward_dynamics(self, action, dof=True, body_acc=True, cfrc_int=False, cfrc_ext=False, out=None):
        """What `action` would do at every env's current state, the state of info["next_obs"], without advancing it: one
        MuJoCo 2.3.7 mj_forward with ctrl mapped from `action` (float32 [num_envs, action_dim] on the env's device) as step()
        maps it, the env's warm start, parameter-pool row and registered xfrc_applied / qfrc_applied, followed by
        mj_rnePostConstraint. Returns a dict of float32 torch tensors on the env's device, one key per output asked for:
            dof       [num_envs, nq, 3]     qfrc_actuator, qfrc_constraint, qacc of this evaluation (dof_outputs' layout;
                                            for Euler, qacc is the explicit mj_forward one, as there)
            body_acc  [num_envs, nbody, 6]  per body the angular acceleration, then the linear acceleration of its origin
                                            xpos minus gravity, world frame (mj_objectAcceleration; an accelerometer at
                                            xpos reads the linear part rotated into its frame: (0, 0, +9.81) at rest)
            cfrc_int  [num_envs, nbody, 6]  the wrench the parent exerts on the body through the joints between them:
                                            force, then torque about xpos, world frame (MuJoCo's cfrc_int; a force /
                                            torque sensor at the body's joint). Row 0 is zeros
            cfrc_ext  [num_envs, nbody, 6]  the external wrench on the body, contacts plus xfrc_applied, in the same layout
                                            (MuJoCo's cfrc_ext). Row 0 is zeros
        Dof axes are in the qvel layout (`dof_index(joint)`), body axes in the model's body order (`body_index(name)`). A
        non-finite state or action gives that env zero rows. `out`: the dict of an earlier call, filled in place and
        returned (a graph-captured loop then allocates nothing); outputs it lacks are allocated. Changes nothing in the env:
        the next step() is the same, bit for bit, as without this call."""
        eng = self._get_engine()
        n, nq, nb = self.num_envs, self._model.nq, self._model.nbody
        shapes = dict(dof=(n, nq, 3), body_acc=(n, nb, 6), cfrc_int=(n, nb, 6), cfrc_ext=(n, nb, 6))
        want = dict(dof=dof, body_acc=body_acc, cfrc_int=cfrc_int, cfrc_ext=cfrc_ext)
        out, got = self._query_outputs("forward_dynamics", self.FORWARD_OUTPUTS, out, want, shapes, eng.device)
        eng.forward(action, **got)
        return out

    @staticmethod
    def _query_outputs(method, names, out, want, shapes, device):
        """(out, got) of a query with the outputs `names`: `out` is the dict of an earlier `method` call, or None for a new
        one; every output k asked for (want[k] true) that it lacks is allocated into it, float32 of shapes[k] on `device`.
        got[k] is out[k] when asked for, else None."""
        import torch
        if out is None:
            out = {}
        elif not isinstance(out, dict):
            raise ValueError("out must be the dict of an earlier %s() call" % method)
        for k in names:
            if want[k] and out.get(k) is None:
                out[k] = torch.empty(shapes[k], dtype=torch.float32, device=device)
        return out, {k: out[k] if want[k] else None for k in names}

    # ---------------------------------------------------------------------------------------------------
    # ray casting (MuJoCo's mj_ray, include/locosim.h locosim_ray) and cameras built on it
    # ---------------------------------------------------------------------------------------------------
    RAY_MODES = dict(world=0, body=1, heading=2, track=3)

    def _body_arg(self, body, what):
        if isinstance(body, str):
            return self.body_index(body)
        b = int(body)
        if not 0 <= b < self._model.nbody:
            raise ValueError("%s %r out of range [0, %d)" % (what, body, self._model.nbody))
        return b

    def ray_cast(self, pnt, vec, frame=None, mode="world", exclude_body=None, static=True, dynamic=True, normal=False,
                 out=None):
        """MuJoCo's mj_ray for every env at its current state, the state of info["next_obs"]: the rays pnt + x vec (float32
        torch tensors on the env's device, [n_rays, 3] for the same rays in every env or [num_envs, n_rays, 3] per env)
        against the env's geoms. `mode` says where the rays are given, relative to body `frame` (a name or an index; the
        root body, index 1, when None):
            "world"    world coordinates (`frame` is not used)
            "body"     the body's frame (position and orientation of body_state)
            "heading"  at the body's origin, turned by the yaw of its x axis only (level height scans that turn with it)
            "track"    at the body's origin with the world's axes
        `static` selects the geoms welded to the world (the floor), `dynamic` the robot's; the geoms of body `exclude_body`
        (name or index) are skipped. Returns a dict of tensors on the env's device:
            dist    float32 [num_envs, n_rays]     the first hit in units of |vec| (metres for a unit vec), -1 for none
            geom    int32 [num_envs, n_rays]       its geom (`geom_index`, `geom_names`), -1 for none
            normal  float32 [num_envs, n_rays, 3]  (normal=True) the unit outward surface normal there, world frame
        Primitives follow MuJoCo 2.3.7 (one-sided planes; a ray that starts inside a geom reports where it leaves it); a
        mesh is hit on the convex hull of its vertices, the shape the engine collides with. A non-finite state gives that
        env -1. `out`: the dict of an earlier call, filled in place (a graph-captured loop then allocates nothing). Changes
        nothing in the env."""
        import torch
        from ..engine import RAY_STATIC, RAY_DYNAMIC, RAY_PER_ENV
        eng = self._get_engine()
        if mode not in self.RAY_MODES:
            raise ValueError("mode must be one of %s" % ", ".join(self.RAY_MODES))
        fb = 0 if mode == "world" else (1 if frame is None else self._body_arg(frame, "frame"))
        ex = -1 if exclude_body is None else self._body_arg(exclude_body, "exclude_body")
        if not isinstance(pnt, torch.Tensor) or pnt.dim() not in (2, 3):
            raise ValueError("pnt must be a float32 torch tensor [n_rays, 3] or [num_envs, n_rays, 3]")
        flags = (RAY_STATIC if static else 0) | (RAY_DYNAMIC if dynamic else 0) | (RAY_PER_ENV if pnt.dim() == 3 else 0)
        n, r = self.num_envs, int(pnt.shape[-2])
        if out is None:
            out = {}
        elif not isinstance(out, dict):
            raise ValueError("out must be the dict of an earlier ray_cast() call")
        shapes = dict(dist=((n, r), torch.float32), geom=((n, r), torch.int32), normal=((n, r, 3), torch.float32))
        for k, (shape, dtype) in shapes.items():
            if (k != "normal" or normal) and (out.get(k) is None or tuple(out[k].shape) != shape):
                out[k] = torch.empty(shape, dtype=dtype, device=eng.device)
        eng.ray(pnt, vec, out["dist"], out["geom"], out["normal"] if normal else None, frame=self.RAY_MODES[mode],
                frame_body=fb, exclude_body=ex, flags=flags)
        return out

    def camera(self, width, height, fovy=45.0, mode="follow", body=None, distance=3.5, elevation=-20.0, azimuth=90.0,
               pos=None, quat=None, normal=False, out=None):
        """Depth and segmentation images of every env from one pinhole camera (one ray per pixel, row-major, pixel (0, 0)
        at the top left; `fovy` in degrees is the angle between the top and bottom image edges):
            "follow"  looks at the origin of `body` (the root when None) from `distance` metres, at `elevation` and
                      `azimuth` degrees (MuJoCo's free camera: elevation < 0 looks down), with the world's axes: the
                      camera_params["follow"] of the reference's viewer
            "body"    fixed to `body` at `pos` (3) with orientation `quat` (w x y z) in its frame, looking along the
                      camera frame's -z with y up (MuJoCo's camera convention): an egocentric camera
        Returns a dict of tensors on the env's device:
            depth   float32 [num_envs, height, width]     distance along the optical axis (metres), inf where nothing is hit
            geom    int32 [num_envs, height, width]       the geom seen, -1 for none
            body    int32 [num_envs, height, width]       its body (`body_index`), -1 for none
            normal  float32 [num_envs, height, width, 3]  (normal=True) unit surface normal, world frame
        and the ray set it cast: pnt / vec (the rays in the query frame, vec of unit length), dist (metres along each ray,
        -1 for none). `out`: the dict of an earlier call with
        the same arguments, filled in place."""
        import math
        import torch
        eng = self._get_engine()
        W, H = int(width), int(height)
        if W < 1 or H < 1:
            raise ValueError("width and height must be positive")
        if mode not in ("follow", "body"):
            raise ValueError('mode must be "follow" or "body"')
        b = 1 if body is None else self._body_arg(body, "body")
        dev = eng.device
        if out is None or out.get("_key") != (W, H, fovy, mode, b, distance, elevation, azimuth, str(pos), str(quat)):
            out = {} if out is None else out
            t = math.tan(math.radians(float(fovy)) / 2)
            jj, ii = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64),
                                    indexing="ij")
            u = (ii + 0.5 - W / 2) / (H / 2) * t
            v = (H / 2 - jj - 0.5) / (H / 2) * t
            if mode == "follow":
                az, el = math.radians(float(azimuth)), math.radians(float(elevation))
                fwd = torch.tensor([math.cos(el) * math.cos(az), math.cos(el) * math.sin(az), math.sin(el)],
                                   dtype=torch.float64)
                up = torch.tensor([-math.sin(el) * math.cos(az), -math.sin(el) * math.sin(az), math.cos(el)],
                                  dtype=torch.float64)
                origin = -float(distance) * fwd
            else:
                from ..mjcf import quat_to_mat
                R = torch.tensor(np.asarray(quat_to_mat(np.asarray([1.0, 0, 0, 0] if quat is None else quat,
                                                                   dtype=np.float64))), dtype=torch.float64)
                fwd, up = -R[:, 2], R[:, 1]
                origin = torch.tensor([0.0, 0, 0] if pos is None else [float(x) for x in pos], dtype=torch.float64)
            right = torch.linalg.cross(fwd, up)
            d = fwd + u[..., None] * right + v[..., None] * up
            d = d / d.norm(dim=-1, keepdim=True)
            out["vec"] = d.reshape(-1, 3).to(torch.float32).to(dev)
            out["pnt"] = origin.expand(H * W, 3).to(torch.float32).contiguous().to(dev)
            out["_cos"] = (d @ fwd).to(torch.float32).reshape(H, W).to(dev)
            out["_key"] = (W, H, fovy, mode, b, distance, elevation, azimuth, str(pos), str(quat))
            out.pop("_rays", None)
        rays = self.ray_cast(out["pnt"], out["vec"], frame=b, mode="track" if mode == "follow" else "body", normal=normal,
                             out=out.get("_rays"))
        out["_rays"] = rays
        n = self.num_envs
        dist, geom = rays["dist"].view(n, H, W), rays["geom"].view(n, H, W)
        if out.get("_bodyid") is None:
            out["_bodyid"] = torch.tensor(np.asarray(self._model.geom_bodyid), dtype=torch.int32, device=dev)
        out["dist"], out["geom"] = dist, geom
        out["depth"] = torch.where(dist >= 0, dist * out["_cos"], torch.full_like(dist, float("inf")))
        out["body"] = torch.where(geom >= 0, out["_bodyid"][geom.clamp(min=0).long()], geom)
        if normal:
            out["normal"] = rays["normal"].view(n, H, W, 3)
        return out

    def _body1_origin(self, env):
        """World position of body 1 (the root) of env `env` at its stored state, from its own joints (kin_body of the
        engine's kinematics in fp64 on the host): where render() puts the floor's checker squares."""
        from ..mjcf import quat_to_mat
        m = self._model
        q = self._get_engine().get_state()[0][int(env)].double().cpu().numpy()
        pos, quat = np.asarray(m.body_pos[1], dtype=np.float64).copy(), np.asarray(m.body_quat[1], dtype=np.float64)
        R = np.asarray(quat_to_mat(quat))
        for j in range(m.body_jntadr[1], m.body_jntadr[1] + m.body_jntnum[1]):
            x = q[j] - m.qpos0[j]
            axis, anchor = R @ np.asarray(m.jnt_axis[j]), pos + R @ np.asarray(m.jnt_pos[j])
            if m.jnt_type[j] == mjcf.JNT_SLIDE:
                pos = pos + axis * x
            else:
                c, s = np.cos(x), np.sin(x)
                K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
                Rj = np.eye(3) + s * K + (1 - c) * K @ K
                pos, R = anchor + Rj @ (pos - anchor), Rj @ R
        return pos

    # ---------------------------------------------------------------------------------------------------
    # saved states (MuJoCo's mj_copyData for a batch, include/locosim.h locosim_save_state / locosim_load_state)
    # ---------------------------------------------------------------------------------------------------
    def save_state(self, out=None):
        """Every env's whole simulation state as one int32 torch tensor [num_envs, W] on the env's device, one row per env:
        qpos, qvel, the solver's warm start, the goal, the reset counter of the env's random stream, its parameter-pool row
        (domain randomisation, the carried weight), trajectory cursor, episode length and return, rotation angle, and the
        observation it acts on next (`engine.state_layout(nq, obs_dim)` names the words). `out`: a tensor of an earlier call,
        filled in place (a graph-captured loop then allocates nothing). Rows load into any env of an env of the same task
        (`load_state`); this env's shards and MixedBatch members included. Call after reset()."""
        if self._obs is None:
            raise RuntimeError("save_state() before the first reset(): there is no state to save")
        eng = self._get_engine()
        return eng.save_state(self._obs_tensor(eng), out)

    def load_state(self, state, index=None):
        """Put envs back into saved states: env i takes row index[i] of `state` (int32 [M, W] from `save_state`, any M;
        `index` int32 [num_envs] on the env's device, or None for row i, then M must be num_envs). A negative index, one
        >= M, or a row saved by an env of another task leaves the env untouched. Returns the observation to act on next,
        as reset() does (untouched envs' rows unchanged). Loading a row back into the env it came from and replaying the
        same actions gives the same results bit for bit, auto-resets included. A loaded env keeps its own id: its next
        reset draws from its own random stream, so envs forked from one row are identical until their first reset.
        Not restored: `xfrc_applied` / `qfrc_applied` (index them with the same rows), the host-side state of a custom
        reward callback and, in the drop-in single-env mode, the host-side trajectory sampler and numpy random state.
        Call after reset()."""
        if self._obs is None:
            raise RuntimeError("load_state() before the first reset(): reset first, so that envs not loaded have an observation")
        eng = self._get_engine()
        obs = self._obs_tensor(eng)
        if obs.data_ptr() != eng.next_obs.data_ptr():
            eng.next_obs.copy_(obs)
        eng.load_state(state, index, obs_out=eng.next_obs)
        if not self.batched:
            self._obs = eng.next_obs[0].double().cpu().numpy()
            return self._obs.copy()
        self._obs = eng.next_obs.clone() if self._copy_outputs else eng.next_obs
        return self._obs

    def _obs_tensor(self, eng):
        """The observation the env acts on next as a float32 [num_envs, obs_dim] tensor on the engine's device."""
        if self.batched:
            return self._obs
        import torch
        return torch.tensor(self._obs, dtype=torch.float32, device=eng.device).reshape(1, -1)

    # ---------------------------------------------------------------------------------------------------
    # the hot path
    # ---------------------------------------------------------------------------------------------------
    def reward(self, state, action, next_state, absorbing):
        return self._reward_function(state, action, next_state, absorbing)

    def _state_from_obs(self, obs):
        """Observation(s) -> (qpos, qvel) [n, nq] (root x / y = 0), goal features [n, n_goal] or None.
        Reference: LocoEnv._init_sim_from_obs + set_sim_state (base.py:478-497,633-654)."""
        obs = np.atleast_2d(np.asarray(obs, dtype=np.float64))
        types, idxs = self._obs_sources()
        assert obs.shape[1] >= len(types), "observation shorter than the observation specification"
        nq = self._model.nq
        q, v = np.zeros((len(obs), nq)), np.zeros((len(obs), nq))
        goal = np.zeros((len(obs), 4))
        for k, (t, i) in enumerate(zip(types, idxs)):
            if t == OBS_QPOS:
                q[:, i] = obs[:, k]
            elif t == OBS_QVEL:
                v[:, i] = obs[:, k]
            elif t == OBS_GOAL:
                goal[:, i] = obs[:, k]
        return q, v, (goal if self._n_goal() else None)

    def _reset_from_obs(self, eng, obs):
        import torch
        if torch.is_tensor(obs):
            obs = obs.detach().cpu().numpy()
        q, v, goal = self._state_from_obs(obs)
        assert len(q) == self.num_envs, "reset(obs): one observation per env"
        if len(self._models) > 1:
            raise NotImplementedError("reset(obs=...) of a multi-model env")
        eng.reset()                                   # episode bookkeeping (counters, parameter-pool row, foot forces)
        f = lambda a: torch.tensor(a, dtype=torch.float32, device=eng.device).contiguous()
        eng.set_state(f(q), f(v))
        if goal is not None:
            eng.set_goal(f(goal))
        out = f(np.atleast_2d(np.asarray(obs, dtype=np.float64))[:, :eng.obs_dim])
        if out.shape[1] < eng.obs_dim:                # foot forces / per-model features: zero / unchanged after a reset
            out = torch.cat([out, eng.next_obs[:, out.shape[1]:]], dim=1)
        eng.next_obs.copy_(out)
        return eng.next_obs

    def reset(self, obs=None):
        eng = self._get_engine()
        import torch
        self._reward_function.reset_state()
        if obs is None:
            # argument checks of the reference's setup() (base.py:220-225)
            if self.trajectories is None and self._random_start:
                raise ValueError("Random start not possible without trajectory data.")
            if self.trajectories is None and self._init_step_no is not None:
                raise ValueError("Setting an initial step is not possible without trajectory data.")
            if self._init_step_no is not None and self._random_start:
                raise ValueError("Either use a random start or set an initial step, not both.")
        if not self.batched:
            # reference semantics incl. the legacy global numpy RNG draw order (base.py:187-191, trajectory.py:253-259)
            model_no = np.random.randint(0, len(self._models))
            self._current_model_idx = model_no
            if obs is not None:
                out = self._reset_from_obs(eng, obs)
                self._obs = out[0].double().cpu().numpy()
                return self._obs.copy()
            if self._random_start:
                sample = self.trajectories.reset_trajectory()
            elif self._init_step_no is not None:
                T, n_traj = self.trajectories.trajectory_length, self.trajectories.number_of_trajectories
                assert self._init_step_no <= T * n_traj
                sample = self.trajectories.reset_trajectory(int(self._init_step_no % T), int(self._init_step_no / T))
            else:
                sample = self.trajectories.reset_trajectory(substep_no=0)
            traj_no, step_no = self.trajectories.traj_no, self.trajectories.subtraj_step_no
            t = torch.tensor([traj_no], dtype=torch.int32, device=eng.device)
            s = torch.tensor([step_no], dtype=torch.int32, device=eng.device)
            r = torch.tensor([model_no], dtype=torch.int32, device=eng.device) if len(self._models) > 1 else None
            ang = self._reset_rotation_angle()
            ang = None if ang is None else torch.tensor([ang], dtype=torch.float32, device=eng.device)
            out = eng.reset(traj_no=t, step_no=s, pool_row=r, rot_angle=ang)
            self._obs = out[0].double().cpu().numpy()
            return self._obs.copy()
        if obs is not None:
            out = self._reset_from_obs(eng, obs)
        else:
            out = eng.reset()
        self._obs = out.clone() if self._copy_outputs else out
        return self._obs

    def set_launch_geometry(self, warps_per_block):
        """Envs (= warps) per block of the step kernel: None = the engine's choice, -1 = always the largest block, k = k.
        Scheduling only. The engine is rebuilt (state lost): call before reset()."""
        self._warps_per_block = warps_per_block
        if getattr(self, "_engine", None) is not None:
            self._engine.close() if hasattr(self._engine, "close") else None
            self._engine = None

    def _reset_rotation_angle(self):
        """Drop-in single-env reset: host-drawn rotation angle of setup_random_rot envs (None: env has no such option)."""
        return None

    def step(self, action):
        eng = self._get_engine()
        import torch
        if not self.batched:
            a = torch.as_tensor(np.asarray(action, dtype=np.float32).reshape(1, -1), device=eng.device)
            obs, reward, done, _ = eng.step(a.contiguous(), auto_reset=False, want_next_obs=False)
            cur = obs[0].double().cpu().numpy()
            flags = int(done[0].item())
            absorbing = bool(flags & DONE_ABSORBING)
            if self._reward_type == "custom":
                r = self._reward_function(self._obs, np.asarray(action), cur, absorbing)
            else:
                r = float(reward[0].item())
            self._obs = cur
            # (no auto-reset in this mode: a truncated episode is reset by the caller, as in the reference)
            return cur.copy(), r, absorbing, ({"truncated": bool(flags & DONE_TRUNCATED)} if self.time_limited else {})
        if action.dtype != torch.float32:
            action = action.float()
        prev = self._obs
        if self._reward_type == "custom" and not self._copy_outputs and prev is not None:
            prev = prev.clone()          # the engine is about to overwrite the buffer `prev` is a view of
        obs, reward, done, next_obs = eng.step(action.contiguous(), auto_reset=True)
        if self._copy_outputs:
            packed = eng.packed_out.clone()
            obs, reward, done = eng.views_of(packed)
            next_obs = next_obs.clone()
        info = {"next_obs": next_obs}
        if self._reward_type == "custom":
            # CustomReward(state, action, next_state): `state` is the observation the action was taken in (base.py:170-176)
            cb = self._reward_function._reward_callback
            reward = cb(prev, action, obs) if cb is not None else torch.zeros_like(reward)
        self._obs = next_obs
        if self.time_limited:
            # `done` keeps its meaning (absorbing); the last finished episode's length and return are valid where
            # done | truncated (the return sums the ENGINE's rewards: 0 under reward_type="custom")
            done, info["truncated"] = split_done(done)
            _, _, info["episode_length"], info["episode_return"] = eng.episode_stats()
            return obs, reward, done, info
        return obs, reward, done.view(torch.bool), info      # (0/1 bytes reinterpreted, no kernel)

    def is_absorbing(self, obs):
        return self._has_fallen(obs) if self._use_absorbing_states else False

    def stop(self):
        pass

    def render(self, record=False, env=0):
        """A frame of env `env` from the follow camera, shaded in torch from one `camera()` call: a flat colour per body with
        Lambert shading on the surface normal, a checker floor, and a sky colour where nothing is hit. Returns uint8 numpy
        [width, height, 3], the layout of the reference's render(True) (GymnasiumWrapper swaps it to [height, width, 3]).
        The camera is camera_params["follow"] (distance, elevation, azimuth in degrees, looking at the root body), else
        distance 3.5, elevation -20, azimuth 90; the size is the width / height keyword arguments of the env, else 640 x
        480. The engine is headless: the frame is returned whether or not `record` is set, and nothing is displayed.
        Textures, visual-only geoms and shadows are not drawn. The query casts the camera's rays for every env of the
        batch, so its cost grows with num_envs."""
        import torch
        if not 0 <= int(env) < self.num_envs:
            raise ValueError("env %r out of range [0, %d)" % (env, self.num_envs))
        follow = dict(distance=3.5, elevation=-20.0, azimuth=90.0)
        follow.update(self._camera_params.get("follow", {}))
        W, H = self._render_size
        cam = self.camera(W, H, mode="follow", distance=follow["distance"], elevation=follow["elevation"],
                          azimuth=follow["azimuth"], normal=True)
        i = int(env)
        geom, body, nrm = cam["geom"][i], cam["body"][i], cam["normal"][i]
        dirs = cam["vec"].view(H, W, 3)
        hit = geom >= 0
        # sky: lighter towards the horizon
        up = dirs[..., 2].clamp(-1, 1)
        sky = torch.stack([0.55 + 0.25 * (1 - up), 0.7 + 0.2 * (1 - up), 0.95 + 0.0 * up], dim=-1)
        # flat body colours from a fixed palette; the floor (static geoms) as a 0.5 m checker
        palette = torch.tensor([[0.85, 0.45, 0.25], [0.3, 0.55, 0.85], [0.9, 0.8, 0.3], [0.45, 0.75, 0.4],
                                [0.75, 0.4, 0.7], [0.4, 0.75, 0.75], [0.85, 0.6, 0.6], [0.6, 0.6, 0.85]],
                               device=geom.device)
        base = palette[body.clamp(min=0) % len(palette)]
        eye = torch.as_tensor(self._body1_origin(i), dtype=torch.float32, device=geom.device) + cam["pnt"][0]
        point = eye + cam["dist"][i].clamp(min=0)[..., None] * dirs
        checker = ((torch.floor(point[..., 0] / 0.5) + torch.floor(point[..., 1] / 0.5)) % 2)[..., None]
        floor = 0.55 + 0.25 * checker.expand(-1, -1, 3)
        base = torch.where((body == 0)[..., None], floor, base)
        sun = torch.tensor([0.3, 0.2, 0.93], device=geom.device)
        sun = sun / sun.norm()
        lambert = (0.35 + 0.45 * (nrm @ sun).clamp(min=0) + 0.2 * (-(nrm * dirs).sum(-1)).clamp(min=0))[..., None]
        rgb = torch.where(hit[..., None], base * lambert, sky).clamp(0, 1)
        return (rgb * 255).round().to(torch.uint8).transpose(0, 1).contiguous().cpu().numpy()

    # ---------------------------------------------------------------------------------------------------
    # observation bookkeeping (reference: base.py:257-276, 729-775)
    # ---------------------------------------------------------------------------------------------------
    def get_kinematic_obs_mask(self):
        return np.arange(len(self.obs_helper.observation_spec) - 2)

    def get_obs_idx(self, key):
        return [i - 2 for i in self.obs_helper.obs_idx_map[key]]

    def _get_idx(self, keys):
        if type(keys) != list:
            keys = [keys]
        return np.concatenate([self.obs_helper.obs_idx_map[k] for k in keys]) - 2

    def _get_from_obs(self, obs, keys):
        obs = np.concatenate([[0.0, 0.0], obs])
        if type(keys) != list:
            keys = [keys]
        return np.concatenate([self.obs_helper.get_from_obs(obs, k) for k in keys])

    def _get_observation_space(self):
        lo, hi = self.info.observation_space.low[2:], self.info.observation_space.high[2:]
        return self._append_grf_space(lo, hi)

    def _append_grf_space(self, lo, hi):
        if self._use_foot_forces:      # base.py:576-580
            n = self._get_grf_size()
            lo, hi = np.concatenate([lo, -np.ones(n) * np.inf]), np.concatenate([hi, np.ones(n) * np.inf])
        return lo, hi

    @staticmethod
    def _get_grf_size():
        return 12

    def _grf_group_names(self):
        """Foot groups in the order of `_get_ground_forces` (base.py:667-679)."""
        return ["foot_r", "front_foot_r", "foot_l", "front_foot_l"]

    def _grf_spec(self):
        """(n_groups, per-geom group id) for the engine; the floor group is matched against every foot group."""
        if not self._use_foot_forces:
            return 0, None
        groups = dict(self._collision_groups)
        names = self._grf_group_names()
        assert 3 * len(names) == self._get_grf_size()
        gid = -np.ones(self._model.ngeom, dtype=np.int32)
        for g in groups["floor"]:
            gid[self._model.geom_id(g)] = GRF_FLOOR
        for k, name in enumerate(names):
            for g in groups[name]:
                gid[self._model.geom_id(g)] = k
        return len(names), gid

    def _create_observation(self, obs):
        return np.concatenate([obs[2:]]).flatten()

    # hidable parts of the observation, in observation order (POMDP masks; base_robot_humanoid.py:38-90,
    # base_humanoid_4_ages.py:187-241)
    _hidable_obs = ("positions", "velocities", "foot_forces")

    def _len_qpos_qvel(self):
        spec = self.obs_helper.observation_spec
        n_pos = sum(1 for _, _, ot in spec if ot == ObservationType.JOINT_POS)
        n_vel = sum(1 for _, _, ot in spec if ot == ObservationType.JOINT_VEL)
        return n_pos, n_vel

    def get_mask(self, obs_to_hide):
        """Boolean mask over the observation: False for the parts named in `obs_to_hide` ("positions", "velocities",
        "foot_forces", and per env "weight" / "env_type")."""
        if type(obs_to_hide) == str:
            obs_to_hide = (obs_to_hide,)
        assert all(x in self._hidable_obs for x in obs_to_hide), "Some of the observations you want to hide are not" \
                                                                 "supported. Valid observations to hide are %s." \
                                                                 % (self._hidable_obs,)
        pos_dim, vel_dim = self._len_qpos_qvel()
        mask = [np.full(pos_dim - 2, "positions" not in obs_to_hide), np.full(vel_dim, "velocities" not in obs_to_hide)]
        if self._use_foot_forces:
            mask.append(np.full(self._get_grf_size(), "foot_forces" not in obs_to_hide))
        else:
            assert "foot_forces" not in obs_to_hide, "Creating a mask to hide foot forces without activating " \
                                                     "the latter is not allowed."
        n_user = len(self._model_user_features[0])
        if n_user:
            key = self._user_feature_name()
            mask.append(np.full(n_user, key not in obs_to_hide))
        else:
            assert not any(k in obs_to_hide for k in ("weight", "env_type")), \
                "Creating a mask to hide the carried weight / env type without activating the latter is not allowed."
        return np.concatenate(mask).ravel().astype(bool)

    def _user_feature_name(self):
        return "weight"

    def _preprocess_action(self, action):
        return (np.asarray(action).copy() * self.norm_act_delta) + self.norm_act_mean

    def _has_fallen(self, obs, return_err_msg=False):
        fallen, msg = False, ""
        for key, lo, hi in self._has_fallen_terms():
            v = obs[self.get_obs_idx(key)[0]]
            if v < lo or v > hi:
                fallen = True
                msg += "%s condition violated (%f not in [%f, %f]).\n" % (key, v, lo, hi)
        return (fallen, msg) if return_err_msg else fallen

    def _get_reward_function(self, reward_type, reward_params):
        if reward_type == "custom":
            return CustomReward(**reward_params)
        if reward_type == "target_velocity":
            idx = self.get_obs_idx("dq_pelvis_tx")
            assert len(idx) == 1
            return TargetVelocityReward(x_vel_idx=idx[0], **reward_params)
        if reward_type == "x_pos":
            idx = self.get_obs_idx("q_pelvis_tx")
            assert len(idx) == 1
            return PosReward(pos_idx=idx[0])
        if reward_type is None or reward_type == "tracking":      # tracking: evaluated in the kernel only (no host functor)
            return NoReward()
        raise NotImplementedError("The specified reward has not been implemented: %s" % reward_type)

    # ---------------------------------------------------------------------------------------------------
    # datasets / replay (reference: base.py:278-386)
    # ---------------------------------------------------------------------------------------------------
    def create_dataset_device(self):
        """`create_dataset()` built ON the device from the reset table that already lives in HBM: dict of torch.cuda float32
        tensors (states / next_states [n, obs_dim] in observation layout, absorbing / last [n]); same content as the host
        `create_dataset()` with the env's default ignore keys (reference: base.py:278-312, utils/trajectory.py:104-151)."""
        import torch
        states, nxt, last = self._get_engine().create_dataset()
        return dict(states=states, next_states=nxt, absorbing=torch.zeros_like(last), last=last)

    def create_dataset(self, ignore_keys=None):
        if self._dataset is None:
            if self.trajectories is None:
                raise ValueError("No trajectory was passed to the environment. To create a dataset pass a trajectory "
                                 "first.")
            dataset = self.trajectories.create_dataset(ignore_keys=ignore_keys)
            for state in dataset["states"]:
                fallen, msg = self._has_fallen(state, return_err_msg=True)
                if fallen:
                    raise ValueError("Some of the states in the created dataset are terminal states. This should not "
                                     "happen.\n\nViolations:\n" + msg)
            self._dataset = deepcopy(dataset)
            return dataset
        return deepcopy(self._dataset)

    def play_trajectory(self, n_episodes=None, n_steps_per_episode=None, render=False, record=False,
                        recorder_params=None):
        """Kinematic replay (no physics is advanced in the reference either: base.py:314-386)."""
        assert self.trajectories is not None
        if render or record:
            raise NotImplementedError("play_trajectory(render=True / record=True) needs a viewer and a video writer, which "
                                      "this headless engine does not have: call render() after each step instead")
        big = np.iinfo(np.int32).max
        n_episodes = big if n_episodes is None else n_episodes
        n_steps_per_episode = big if n_steps_per_episode is None else n_steps_per_episode
        self.trajectories.reset_trajectory()
        for _ in range(n_episodes):
            for _ in range(n_steps_per_episode):
                sample = self.trajectories.get_next_sample()
                if sample is None:
                    self.trajectories.reset_trajectory()
                    sample = self.trajectories.get_current_sample()
                obs = self._create_observation(np.concatenate(sample))
                if self._has_fallen(obs):
                    print("Has fallen!")
            self.trajectories.reset_trajectory()

    # ---------------------------------------------------------------------------------------------------
    # interpolation hooks (identity by default, reference: base.py:855-893)
    # ---------------------------------------------------------------------------------------------------
    def _get_interpolate_map_params(self):
        return None

    def _get_interpolate_remap_params(self):
        return None

    @staticmethod
    def _interpolate_map(traj, **interpolate_map_params):
        return np.array(traj)

    @staticmethod
    def _interpolate_remap(traj, **interpolate_remap_params):
        return [obs for obs in traj]

    @staticmethod
    def _delete_from_xml_handle(xml_handle, joints_to_remove, motors_to_remove, equ_constraints):
        return xml_handle.delete(joints_to_remove, motors_to_remove, equ_constraints)

    @property
    def xml_handle(self):
        return self._xml_handles[0]

    @property
    def xml_handles(self):
        return self._xml_handles

    # ---------------------------------------------------------------------------------------------------
    # registry / factory (reference: base.py:820-832, 950-967; mushroom Environment.make)
    # ---------------------------------------------------------------------------------------------------
    @classmethod
    def register(cls):
        LocoEnv._registered_envs[cls.__name__] = cls

    @staticmethod
    def list_registered_loco_mujoco():
        return list(LocoEnv._registered_envs.keys())

    @staticmethod
    def make(env_name, *args, **kwargs):
        """`LocoEnv.make("UnitreeA1.simple.real", num_envs=4096)`: dotted id -> env class .generate(*id_parts)."""
        if "." in env_name:
            parts = env_name.split(".")
            env_name, args = parts[0], tuple(parts[1:]) + tuple(args)
        if env_name not in LocoEnv._registered_envs:
            raise KeyError("unknown environment %r; registered: %s" % (env_name, LocoEnv.list_registered_loco_mujoco()))
        env = LocoEnv._registered_envs[env_name]
        return env.generate(*args, **kwargs) if hasattr(env, "generate") else env(*args, **kwargs)

    @classmethod
    def get_all_task_names(cls):
        names = []
        for e in cls.list_registered_loco_mujoco():
            env = cls._registered_envs[e]
            for conf in env.valid_task_confs.get_all_combinations():
                names.append(".".join([env.__name__] + list(conf.values())))
        return names


class _ProcessedTrajectory(Trajectory):
    """Trajectory restored from already-interpolated arrays (bundled assets; see tools/build_assets.py)."""

    def __init__(self, d):
        self.keys = [str(k) for k in d["keys"]]
        self.trajectories = [np.asarray(d["traj_%d" % i]) for i in range(len(self.keys))]
        self.split_points = np.asarray(d["split_points"])
        self._traj_info = None
        self.traj_dt = self.control_dt = float(d["control_dt"])
        self.subtraj_step_no = 0
        self.traj_no = 0
        self.subtraj = self._get_subtraj(self.traj_no)

    def to_dict(self):
        d = dict(keys=np.array(self.keys), split_points=self.split_points, control_dt=self.control_dt)
        for i, t in enumerate(self.trajectories):
            d["traj_%d" % i] = t
        return d


def processed_trajectory_dict(traj):
    d = dict(keys=np.array(traj.keys), split_points=np.asarray(traj.split_points), control_dt=traj.control_dt)
    for i, t in enumerate(traj.trajectories):
        d["traj_%d" % i] = t
    return d


class ValidTaskConf:
    """All valid task configurations of an environment (reference: base.py:972-1041)."""

    def __init__(self, tasks=None, modes=None, data_types=None, non_combinable=None):
        self.tasks, self.modes, self.data_types, self.non_combinable = tasks, modes, data_types, non_combinable
        if non_combinable is not None:
            for nc in non_combinable:
                assert len(nc) == 3

    def get_all(self):
        return deepcopy(self.tasks), deepcopy(self.modes), deepcopy(self.data_types), deepcopy(self.non_combinable)

    def get_all_combinations(self):
        confs = []
        for t, m, dt in product(self.tasks or [None], self.modes or [None], self.data_types or [None]):
            conf = {}
            if t is not None:
                conf["task"] = t
            if m is not None:
                conf["mode"] = m
            if dt is not None:
                conf["data_type"] = dt
            if self.non_combinable is not None:
                # (reference quirk kept: a conf is appended once per non-combinable rule it does not match)
                for bad_t, bad_m, bad_dt in self.non_combinable:
                    if not ((t == bad_t or bad_t is None) and (m == bad_m or bad_m is None) and
                            (dt == bad_dt or bad_dt is None)):
                        confs.append(conf)
            else:
                confs.append(conf)
        return confs
