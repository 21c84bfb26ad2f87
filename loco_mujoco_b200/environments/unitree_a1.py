"""
UnitreeA1 (tasks simple / hard, real dataset) on the batched CUDA engine.
Mirrors /root/reference/loco_mujoco/environments/quadrupeds/unitreeA1.py:21-928 : observation / action
specification (:778-854), goal features (:454-476, :722-753), VelocityVectorReward wiring (:478-501),
_has_fallen (:503-536), trajectory (un)mapping for interpolation (:856-928), generate() (:622-710).
"""
import os
import warnings
from copy import deepcopy

import numpy as np

from .. import mjcf
from ..task import OBS_GOAL, REWARD_VELOCITY_VECTOR
from ..utils.checks import check_validity_task_mode_dataset
from ..utils.goals import GoalDirectionVelocity
from ..utils.math import mat2angle_xy, angle2mat_xy, transform_angle_2pi, rotate_obs
from ..utils.reward import VelocityVectorReward
from .base import LocoEnv, ObservationType, ValidTaskConf, reference_data_root, ASSET_DIR, asset_path

ACTION_MODES = ("torque", "position", "position_difference")


def _check_action_mode(action_mode):
    if action_mode not in ACTION_MODES:
        raise ValueError("action_mode must be one of %s, not %r" % (", ".join(map(repr, ACTION_MODES)), action_mode))


_LEGS = ["FR", "FL", "RR", "RL"]
_TRUNK = ["trunk_tx", "trunk_ty", "trunk_tz", "trunk_list", "trunk_tilt", "trunk_rotation"]


class UnitreeA1(LocoEnv):
    valid_task_confs = ValidTaskConf(tasks=["simple", "hard"], data_types=["real", "perfect"])
    _terrain_supported = True

    def __init__(self, action_mode="torque", setup_random_rot=False, default_target_velocity=0.5, camera_params=None,
                 **kwargs):
        # "torque": twelve motors (gear 34, ctrl in [-1, 1]); "position" / "position_difference": twelve PD position
        # actuators (kp 100, force clamped to +-33.5), whose ctrlrange is each joint's range, so the normalised action +-1
        # is a target angle at the ends of that range (unitreeA1.py:196-218). "position_difference" is the same model and
        # the same controller: the reference stores the mode and reads it nowhere else.
        _check_action_mode(action_mode)
        self._action_mode = action_mode
        action_spec = self._get_action_specification()
        observation_spec = self._get_observation_specification()
        observation_spec.append(("dir_arrow", "dir_arrow", ObservationType.SITE_ROT))
        self.setup_random_rot = setup_random_rot
        self._goal = GoalDirectionVelocity()
        self._goal.set_goal(0.0, default_target_velocity)
        if kwargs.get("compiled_model") is None:
            root = reference_data_root()
            if root is None:
                raise FileNotFoundError("loco_mujoco model data not found (set LOCO_MUJOCO_PATH) and no compiled "
                                        "model supplied")
            xml = "unitree_a1_torque.xml" if action_mode == "torque" else "unitree_a1_position.xml"
            xml_handle = mjcf.XmlHandle(os.path.join(root, "environments", "data", "quadrupeds", xml))
            # (the reference also attaches a mass-less `dir_arrow` marker body + two sites to the trunk,
            #  unitreeA1.py:755-776: visualisation only, no geoms, no inertia -> not part of the physics model)
        else:
            xml_handle = None
        collision_groups = [("floor", ["floor"]), ("foot_FR", ["FR_foot"]), ("foot_FL", ["FL_foot"]),
                            ("foot_RR", ["RR_foot"]), ("foot_RL", ["RL_foot"])]      # unitreeA1.py:223-227
        if camera_params is None:
            camera_params = dict(follow=dict(distance=3.5, elevation=-20.0, azimuth=90.0))   # unitreeA1.py:239-241
        super().__init__(xml_handle, action_spec, observation_spec, collision_groups, camera_params=camera_params, **kwargs)

    # -- observation layout -------------------------------------------------------------------------------
    def _get_observation_space(self):
        dir_arrow_idx = self._get_idx("dir_arrow")
        lo, hi = self.info.observation_space.low[2:], self.info.observation_space.high[2:]
        lo = np.concatenate([lo[:dir_arrow_idx[0]], [-1, -1], [-np.inf]])
        hi = np.concatenate([hi[:dir_arrow_idx[0]], [1, 1], [np.inf]])
        return self._append_grf_space(lo, hi)        # unitreeA1.py:432-439

    def _grf_group_names(self):
        return ["foot_FL", "foot_FR", "foot_RL", "foot_RR"]      # unitreeA1.py:551-562

    def _obs_sources(self):
        spec = self.obs_helper.observation_spec
        save = self.obs_helper.observation_spec
        self.obs_helper.observation_spec = spec[:-1]          # joints only
        types, idxs = super()._obs_sources()
        self.obs_helper.observation_spec = save
        return types + [OBS_GOAL] * 3, idxs + [0, 1, 2]

    def _n_goal(self):
        return 3

    def _random_rot_spec(self):
        # setup_random_rot (unitreeA1.py:270-285): yaw and root (vx, vy) of every reset sample are rotated by a ~ U[0, 2 pi);
        # the goal direction is NOT rotated in the reference (it is read from the un-rotated dir_arrow), kept that way
        if not self.setup_random_rot:
            return None
        return (self._model.joint_id("trunk_rotation"), self._model.joint_id("trunk_tx"), self._model.joint_id("trunk_ty"))

    def _reset_rotation_angle(self):
        # drop-in single-env mode: the reference draws the angle from the legacy numpy stream right after the trajectory
        # sample (unitreeA1.py:269-272, 282-285; only for random_start / the first-sample start, not for init_step_no)
        if self.setup_random_rot and (self._random_start or self._init_step_no is None):
            return np.random.uniform(0, 2 * np.pi)
        return 0.0 if self.setup_random_rot else None

    def _goal_features(self, sample):
        rot_mat = self.trajectories.get_from_sample(sample, "dir_arrow")
        angle = transform_angle_2pi(mat2angle_xy(np.asarray(rot_mat))) - np.pi / 2
        speed = float(np.squeeze(self.trajectories.get_from_sample(sample, "goal_speed")))
        return [np.cos(angle), np.sin(angle), speed]

    @property
    def _goal_velocity_idx(self):
        return 43

    @staticmethod
    def _modify_observation_callback(obs, rot_mat_idx_arrow, goal_velocity_idx):
        angle = transform_angle_2pi(mat2angle_xy(obs[rot_mat_idx_arrow].reshape((3, 3)))) - np.pi / 2
        return np.concatenate([obs[:rot_mat_idx_arrow[0]], [np.cos(angle), np.sin(angle)], [obs[goal_velocity_idx]]])

    def _create_observation(self, obs):
        obs = np.concatenate([obs[2:], [self._goal.get_velocity()]]).flatten()
        return self._modify_observation_callback(obs, self._get_idx("dir_arrow"), self._goal_velocity_idx)

    # -- reward / termination -----------------------------------------------------------------------------
    def _reward_spec(self):
        if self._reward_type == "velocity_vector":
            D = self.info.observation_space.shape[0]
            return REWARD_VELOCITY_VECTOR, [self.get_obs_idx("dq_trunk_tx")[0], self.get_obs_idx("dq_trunk_ty")[0],
                                            D - 3, D - 1], []
        return super()._reward_spec()

    def _get_reward_function(self, reward_type, reward_params):
        if reward_type == "velocity_vector":
            return VelocityVectorReward(x_vel_idx=self.get_obs_idx("dq_trunk_tx")[0],
                                        y_vel_idx=self.get_obs_idx("dq_trunk_ty")[0], angle_idx=[-3, -2],
                                        goal_vel_idx=[-1])
        return super()._get_reward_function(reward_type, reward_params)

    def _has_fallen_terms(self):
        return [("q_trunk_list", -0.2793, 0.2793), ("q_trunk_tilt", -0.192, 0.192), ("q_trunk_tz", -0.24, np.inf)]

    # -- datasets ---------------------------------------------------------------------------------------------
    def create_dataset(self, ignore_keys=None):
        if self._dataset is None:
            if ignore_keys is None:
                ignore_keys = ["q_trunk_tx", "q_trunk_ty"]
            if self.trajectories is None:
                raise ValueError("No trajectory was passed to the environment. To create a dataset pass a trajectory "
                                 "first.")
            params = dict(rot_mat_idx_arrow=self._get_idx("dir_arrow"), goal_velocity_idx=self._goal_velocity_idx)
            dataset = self.trajectories.create_dataset(ignore_keys=ignore_keys,
                                                       state_callback=self._modify_observation_callback,
                                                       state_callback_params=params)
            self._dataset = deepcopy(dataset)
            return dataset
        return deepcopy(self._dataset)

    def get_kinematic_obs_mask(self):
        return np.arange(len(self.obs_helper.observation_spec))

    def _get_relevant_idx_rotation(self):
        keys = self.obs_helper.get_all_observation_keys()
        return keys.index("q_trunk_rotation"), keys.index("dq_trunk_tx"), keys.index("dq_trunk_ty")

    def play_trajectory(self, *args, **kwargs):
        # samples carry the extra goal_speed entry, which is not part of the simulation state
        assert self.trajectories is not None
        n_episodes = kwargs.get("n_episodes") or (args[0] if args else None)
        n_steps = kwargs.get("n_steps_per_episode") or (args[1] if len(args) > 1 else None)
        big = np.iinfo(np.int32).max
        self.trajectories.reset_trajectory()
        for _ in range(big if n_episodes is None else n_episodes):
            for _ in range(big if n_steps is None else n_steps):
                sample = self.trajectories.get_next_sample()
                if sample is None:
                    self.trajectories.reset_trajectory()
                    sample = self.trajectories.get_current_sample()
                self._goal.set_goal(mat2angle_xy(np.asarray(sample[-2])), float(np.squeeze(sample[-1])))
                obs = self._create_observation(np.concatenate(sample[:-1]))
                if self._has_fallen(obs):
                    print("Has fallen!")
            self.trajectories.reset_trajectory()

    # -- interpolation maps -------------------------------------------------------------------------------------
    def _get_interpolate_map_params(self):
        keys = self.get_all_observation_keys()
        return dict(rot_mat_idx=keys.index("dir_arrow"),
                    trunk_orientation_idx=[keys.index("q_trunk_list"), keys.index("q_trunk_tilt"),
                                           keys.index("q_trunk_rotation")])

    def _get_interpolate_remap_params(self):
        keys = self.get_all_observation_keys()
        return dict(angle_idx=keys.index("dir_arrow"),
                    trunk_orientation_idx=[keys.index("q_trunk_list"), keys.index("q_trunk_tilt"),
                                           keys.index("q_trunk_rotation")],
                    position_indices=[keys.index(k) for k in keys if k.startswith("q_")],
                    velocity_indices=[keys.index(k) for k in keys if k.startswith("dq_")], ctrl_dt=self.dt)

    @staticmethod
    def _interpolate_map(traj, **p):
        out = []
        for i, series in enumerate(traj):
            if i == p["rot_mat_idx"]:
                out.append(np.array([mat2angle_xy(mat) for mat in series]))
            elif i in p["trunk_orientation_idx"]:
                out.append(np.unwrap(series))
            else:
                out.append(np.asarray(series))
        return np.array(out)

    @staticmethod
    def _interpolate_remap(traj, **p):
        out = [None] * len(traj)
        for i in range(len(traj)):
            if i == p["angle_idx"]:
                out[i] = np.array([angle2mat_xy(a).reshape(9,) for a in traj[i]])
            elif i in p["trunk_orientation_idx"]:
                out[i] = [transform_angle_2pi(a) for a in traj[i]]
            elif i in p["velocity_indices"]:
                # velocities are re-derived from the interpolated positions (finite differences)
                pos = traj[p["position_indices"][p["velocity_indices"].index(i)]]
                out[i] = [0.0] + list((pos[1:] - pos[:-1]) / p["ctrl_dt"])
            else:
                out[i] = list(traj[i])
        return out

    # -- specification ---------------------------------------------------------------------------------------------
    @staticmethod
    def _get_observation_specification():
        joints = _TRUNK + ["%s_%s_joint" % (l, p) for l in _LEGS for p in ("hip", "thigh", "calf")]
        spec = [("q_" + j, j, ObservationType.JOINT_POS) for j in joints]
        spec += [("dq_" + j, j, ObservationType.JOINT_VEL) for j in joints]
        return spec

    @staticmethod
    def _get_action_specification():
        return ["%s_%s" % (l, p) for l in _LEGS for p in ("hip", "thigh", "calf")]

    @staticmethod
    def generate(task="simple", dataset_type="real", debug=False, **kwargs):
        check_validity_task_mode_dataset(UnitreeA1.__name__, task, None, dataset_type,
                                         *UnitreeA1.valid_task_confs.get_all())
        if dataset_type != "real":
            raise NotImplementedError("perfect datasets are not shipped (network download in the reference)")
        if "reward_type" in kwargs:
            reward_type, reward_params = kwargs.pop("reward_type"), kwargs.pop("reward_params", dict())
        else:
            reward_type, reward_params = "velocity_vector", dict()
        fname = "walk_straight.npz" if task == "simple" else "walk_8_dir.npz"
        root = reference_data_root()
        if root is not None:
            path = os.path.join(root, "datasets", "quadrupeds", "real", fname)
            if debug or not os.path.exists(path):
                if not os.path.exists(path) and not debug:
                    warnings.warn("Datasets not found, falling back to test datasets. Please download and install "
                                  "the datasets to use this environment for imitation learning!")
                path = os.path.join(root, "datasets", "quadrupeds", "real", "mini_datasets", fname)
            mdp = UnitreeA1(reward_type=reward_type, reward_params=reward_params, **kwargs)
            mdp.load_trajectory(dict(traj_path=path, traj_dt=1 / 500.0, control_dt=mdp.dt))
        else:
            from .. import modelpack
            action_mode = kwargs.get("action_mode", "torque")
            if action_mode == "torque":
                path = os.path.join(ASSET_DIR, "UnitreeA1.%s.npz" % task)
            else:
                _check_action_mode(action_mode)      # (an unknown mode is a ValueError, not a missing asset)
                # both position modes share one model, UnitreeA1.<task>+position.npz; never the torque model instead
                path = asset_path("UnitreeA1.%s+position.npz" % task)
                if path is None:
                    raise FileNotFoundError(
                        "no bundled asset for UnitreeA1.%s+position (action_mode=%r): the package bundles the torque "
                        "models; the position models are compiled from a loco_mujoco checkout (set LOCO_MUJOCO_PATH) or "
                        "read from a directory of assets made by tools/build_assets.py (set LOCO_MUJOCO_B200_ASSET_PATH)"
                        % (task, action_mode))
            asset = np.load(path, allow_pickle=False)
            model = modelpack.from_npz_dict({k[6:]: asset[k] for k in asset.files if k.startswith("model_")})
            mdp = UnitreeA1(reward_type=reward_type, reward_params=reward_params, compiled_model=model, **kwargs)
            mdp.load_trajectory(dict(processed={k[5:]: asset[k] for k in asset.files if k.startswith("traj_")}))
        return mdp
