"""
Atlas, Talos (walk) and UnitreeH1 (walk, run), real datasets, on the batched CUDA engine.
Mirrors /root/reference/loco_mujoco/environments/humanoids/base_robot_humanoid.py:12-260 (generate, dataset keys),
atlas.py:275-453,485-598, talos.py:266-466,523-640 and unitreeH1.py:235-296,319-384,447-553 (joint/motor removal,
observation/action specification, _has_fallen windows).
"""
import inspect
import os
import warnings

import numpy as np

from .. import mjcf
from ..utils.checks import check_validity_task_mode_dataset
from .base import LocoEnv, ObservationType, ValidTaskConf, reference_data_root, asset_path

_PELVIS = ["pelvis_tx", "pelvis_tz", "pelvis_ty", "pelvis_tilt", "pelvis_list", "pelvis_rotation"]
_ARMS = ["%s_arm_%s" % (s, j) for s in ("l", "r") for j in ("shz", "shx", "ely", "elx", "wry", "wrx")]
_LEGS = ["%s_%s" % (j, s) for s in ("r", "l") for j in ("hip_flexion", "hip_adduction", "hip_rotation", "knee_angle",
                                                        "ankle_angle")]


class BaseRobotHumanoid(LocoEnv):
    _xml_rel = None
    _mini_dataset = None

    _valid_weights = [0.1, 1.0, 5.0, 10.0]
    _hidable_obs = ("positions", "velocities", "foot_forces", "weight")

    def __init__(self, disable_arms=True, disable_back_joint=True, hold_weight=False, weight_mass=None, **kwargs):
        if hold_weight:
            assert disable_arms is True, "If you want the robot to carry a weight, please disable the arms. " \
                                         "They will be kept fixed."
        self._disable_arms, self._disable_back_joint, self._hold_weight = disable_arms, disable_back_joint, hold_weight
        self._weight_mass = weight_mass
        action_spec = self._get_action_specification()
        observation_spec = self._get_observation_specification()
        joints_to_remove, motors_to_remove, equ = self._get_xml_modifications()
        hide = ["q_" + j for j in joints_to_remove] + ["dq_" + j for j in joints_to_remove]
        observation_spec = [e for e in observation_spec if e[0] not in hide]
        action_spec = [a for a in action_spec if a not in motors_to_remove]
        weights = ([weight_mass] if weight_mass is not None else list(self._valid_weights)) if hold_weight else []
        if kwargs.get("compiled_model") is None:
            root = reference_data_root()
            if root is None:
                raise FileNotFoundError("loco_mujoco model data not found (set LOCO_MUJOCO_PATH)")
            xml_handle = mjcf.XmlHandle(os.path.join(root, "environments", "data", *self._xml_rel))
            xml_handle = self._delete_from_xml_handle(xml_handle, joints_to_remove, motors_to_remove, equ)
            if hold_weight:     # one model per weight (atlas.py:316-331, talos.py:310-322)
                xml_handle = [self._add_weight(xml_handle.copy(), w) for w in weights]
            else:
                xml_handle = self._modify_xml(xml_handle)
        else:
            xml_handle = None
        super().__init__(xml_handle, action_spec, observation_spec, self._collision_groups_spec(), **kwargs)
        if hold_weight:
            assert len(self._models) == len(weights)
            self._model_user_features = [(float(w),) for w in weights]     # observed weight mass

    def _add_weight(self, xml_handle, mass):
        raise NotImplementedError("%s has no carry task" % type(self).__name__)

    def _get_observation_space(self):
        lo, hi = super()._get_observation_space()
        if self._hold_weight:       # base_robot_humanoid.py:100-103
            lo, hi = np.concatenate([lo, [self._valid_weights[0]]]), np.concatenate([hi, [self._valid_weights[-1]]])
        return lo, hi

    def _collision_groups_spec(self):
        # atlas.py:292-296 (4 groups, base-class _get_ground_forces)
        return [("floor", ["floor"]), ("foot_r", ["right_foot_back"]), ("front_foot_r", ["right_foot_front"]),
                ("foot_l", ["left_foot_back"]), ("front_foot_l", ["left_foot_front"])]

    def _modify_xml(self, xml_handle):
        return xml_handle

    def create_dataset(self, ignore_keys=None):
        if ignore_keys is None:
            ignore_keys = ["q_pelvis_tx", "q_pelvis_tz"]
        return super().create_dataset(ignore_keys)

    def _pelvis_terms(self):
        return [("q_pelvis_ty", -0.3, 0.1), ("q_pelvis_tilt", -np.pi / 4.5, np.pi / 12),
                ("q_pelvis_list", -np.pi / 12, np.pi / 8), ("q_pelvis_rotation", -np.pi / 10, np.pi / 10)]

    @classmethod
    def _generate(cls, dataset_stub, task="walk", dataset_type="real", debug=False,
                  clip_trajectory_to_joint_ranges=False, **kwargs):
        check_validity_task_mode_dataset(cls.__name__, task, None, dataset_type, *cls.valid_task_confs.get_all())
        if dataset_type != "real":
            raise NotImplementedError("perfect datasets are not shipped (network download in the reference)")
        if task not in ("walk", "run", "carry"):
            raise NotImplementedError("task %r is not built yet" % task)
        if task == "carry":
            # base_robot_humanoid.py: the carried weight needs the arms fixed (asserted before any asset is looked up)
            assert kwargs.get("disable_arms", True) is True, "If you want the robot to carry a weight, please disable " \
                                                             "the arms. They will be kept fixed."
            kwargs["hold_weight"] = True
        variant = cls.variant_suffix(**kwargs)
        reward_type = kwargs.pop("reward_type", "target_velocity")
        reward_params = kwargs.pop("reward_params", dict(target_velocity=2.5 if task == "run" else 1.25))
        root = reference_data_root()
        if root is not None:
            mdp = cls(reward_type=reward_type, reward_params=reward_params, **kwargs)
            path = os.path.join(root, "datasets", "humanoids", "real", dataset_stub)
            if debug or not os.path.exists(path):
                if not os.path.exists(path) and not debug:
                    warnings.warn("Datasets not found, falling back to test datasets. Please download and install "
                                  "the datasets to use this environment for imitation learning!")
                path = os.path.join(root, "datasets", "humanoids", "real", "mini_datasets", dataset_stub)
            mdp.load_trajectory(dict(traj_path=path, traj_dt=1 / 500.0, control_dt=mdp.dt,
                                     clip_trajectory_to_joint_ranges=clip_trajectory_to_joint_ranges), warn=False)
        else:
            from .. import modelpack
            path = asset_path("%s.%s%s.npz" % (cls.__name__, task, variant))
            if path is None:
                raise FileNotFoundError(
                    "no bundled asset for %s.%s%s (%s): the package bundles the default models; other variants are "
                    "compiled from a loco_mujoco checkout (set LOCO_MUJOCO_PATH) or read from a directory of assets made "
                    "by tools/build_assets.py (set LOCO_MUJOCO_B200_ASSET_PATH)"
                    % (cls.__name__, task, variant,
                       ", ".join("%s=%s" % kv for kv in sorted(cls._variant_kwargs(kwargs).items()))))
            asset = np.load(path, allow_pickle=False)
            n_models = int(asset["n_models"]) if "n_models" in asset.files else 1
            if n_models > 1:
                model = [modelpack.from_npz_dict({k[len("model%d_" % i):]: asset[k] for k in asset.files
                                                  if k.startswith("model%d_" % i)}) for i in range(n_models)]
            else:
                model = modelpack.from_npz_dict({k[6:]: asset[k] for k in asset.files if k.startswith("model_")})
            mdp = cls(reward_type=reward_type, reward_params=reward_params, compiled_model=model, **kwargs)
            mdp.load_trajectory(dict(processed={k[5:]: asset[k] for k in asset.files if k.startswith("traj_")}))
        mdp._task_id = "%s.%s%s" % (cls.__name__, task, variant)
        return mdp

    @classmethod
    def _variant_kwargs(cls, kwargs):
        """The model-variant options of a constructor call, with the class's defaults filled in."""
        params = inspect.signature(cls.__init__).parameters
        return {k: kwargs.get(k, params[k].default) for k in ("disable_arms", "disable_back_joint")}

    @classmethod
    def variant_suffix(cls, **kwargs):
        """Suffix that names a model variant in asset and DR-pool file names: "" for the class's default model, else
        "+arms" / "+back" for a part enabled that the default disables ("-arms" / "-back" for the reverse), e.g.
        Atlas(disable_arms=False, disable_back_joint=False) -> "+arms+back"."""
        params, chosen = inspect.signature(cls.__init__).parameters, cls._variant_kwargs(kwargs)
        suffix = ""
        for key, part in (("disable_arms", "arms"), ("disable_back_joint", "back")):
            if chosen[key] != params[key].default:
                suffix += ("-" if chosen[key] else "+") + part
        return suffix


class Atlas(BaseRobotHumanoid):
    valid_task_confs = ValidTaskConf(tasks=["walk", "carry"], data_types=["real", "perfect"])
    _xml_rel = ("atlas", "atlas.xml")

    def _get_xml_modifications(self):
        joints, motors = [], []
        if self._disable_arms:
            joints += _ARMS
            motors += [j + "_actuator" for j in _ARMS]
        if self._disable_back_joint:
            joints += ["back_bkz", "back_bky", "back_bkx"]
            motors += ["back_bkz_actuator", "back_bky_actuator", "back_bkx_actuator"]
        return joints, motors, []

    def _add_weight(self, h, mass):        # atlas.py:456-482
        w = h.add(h.find("body", "utorso"), "body", name="weight")
        h.add(w, "geom", type="box", size="0.1 0.27 0.1", pos="0.72 0 -0.25", group="0", mass=repr(float(mass)))
        h.find("body", "r_clav").set("quat", "1.0 0.0 -0.35 0.0")
        h.find("body", "l_clav").set("quat", "0.0 -0.35 0.0 1.0")
        return h

    def _has_fallen_terms(self):
        terms = self._pelvis_terms()
        if not self._disable_back_joint:
            terms += [("q_back_bky", -np.pi / 4, np.pi / 10), ("q_back_bkx", -np.pi / 10, np.pi / 10),
                      ("q_back_bkz", -np.pi / 4.5, np.pi / 4.5)]
        return terms

    @staticmethod
    def _get_observation_specification():
        joints = _PELVIS + ["back_bkz", "back_bkx", "back_bky"] + _ARMS + _LEGS
        return [("q_" + j, j, ObservationType.JOINT_POS) for j in joints] + \
               [("dq_" + j, j, ObservationType.JOINT_VEL) for j in joints]

    @staticmethod
    def _get_action_specification():
        return ["back_bkz_actuator", "back_bky_actuator", "back_bkx_actuator"] + [j + "_actuator" for j in _ARMS] + \
               [j + "_actuator" for j in _LEGS]

    @staticmethod
    def generate(task="walk", dataset_type="real", **kwargs):
        return Atlas._generate("02-constspeed_ATLAS.npz", task, dataset_type, **kwargs)


class Talos(BaseRobotHumanoid):
    valid_task_confs = ValidTaskConf(tasks=["walk", "carry"], data_types=["real", "perfect"])
    _xml_rel = ("talos", "talos.xml")

    def __init__(self, disable_arms=True, disable_back_joint=False, hold_weight=False, weight_mass=None, **kwargs):
        super().__init__(disable_arms=disable_arms, disable_back_joint=disable_back_joint, hold_weight=hold_weight,
                         weight_mass=weight_mass, **kwargs)

    def _collision_groups_spec(self):
        return [("floor", ["floor"]), ("foot_r", ["right_foot"]), ("foot_l", ["left_foot"])]

    @staticmethod
    def _get_grf_size():
        return 6

    def _grf_group_names(self):
        return ["foot_r", "foot_l"]

    def _add_weight(self, h, mass):        # talos.py:469-500
        w = h.add(h.find("body", "torso_2_link"), "body", name="weight")
        h.add(w, "geom", type="box", size="0.1 0.25 0.1", pos="0.45 0 -0.20", group="0", mass=repr(float(mass)))
        for name, quat in (("arm_right_4_link", "1.0 0.0 -0.65 0.0"), ("arm_left_4_link", "1.0 0.0 -0.65 0.0"),
                           ("arm_right_6_link", "1.0 0.0 -0.0 1.0"), ("arm_left_6_link", "1.0 0.0 -0.0 1.0")):
            h.find("body", name).set("quat", quat)
        return h

    def _modify_xml(self, xml_handle):
        if self._disable_arms:
            # arms are kept fixed in a reoriented pose (talos.py:503-521)
            for name, quat in _TALOS_ARM_QUATS.items():
                b = xml_handle.find("body", name)
                b.set("quat", " ".join(repr(float(x)) for x in quat))
        return xml_handle

    def _get_xml_modifications(self):
        joints, motors = [], []
        if self._disable_arms:
            joints += _ARMS
            motors += [j + "_actuator" for j in _ARMS]
        if self._disable_back_joint:
            joints += ["back_bkz", "back_bky"]
            motors += ["back_bkz_actuator", "back_bky_actuator"]
        return joints, motors, []

    def _has_fallen_terms(self):
        terms = self._pelvis_terms()
        if not self._disable_back_joint:
            terms += [("q_back_bky", -np.pi / 4, np.pi / 10), ("q_back_bkz", -np.pi / 10, np.pi / 10)]
        return terms

    @staticmethod
    def _get_observation_specification():
        joints = _PELVIS + ["back_bkz", "back_bky"] + _ARMS + _LEGS
        return [("q_" + j, j, ObservationType.JOINT_POS) for j in joints] + \
               [("dq_" + j, j, ObservationType.JOINT_VEL) for j in joints]

    @staticmethod
    def _get_action_specification():
        return ["back_bkz_actuator", "back_bky_actuator"] + [j + "_actuator" for j in _ARMS] + \
               [j + "_actuator" for j in _LEGS]

    @staticmethod
    def generate(task="walk", dataset_type="real", **kwargs):
        return Talos._generate("02-constspeed_TALOS.npz", task, dataset_type, **kwargs)


_TALOS_ARM_QUATS = {"arm_right_4_link": [1.0, 0.0, -0.25, 0.0], "arm_left_4_link": [1.0, 0.0, -0.25, 0.0]}


_H1_ARMS = ["l_arm_shy", "l_arm_shx", "l_arm_shz", "left_elbow", "r_arm_shy", "r_arm_shx", "r_arm_shz", "right_elbow"]
_H1_ARM_QUATS = {"left_shoulder_pitch_link": [1.0, 0.25, 0.1, 0.0], "right_elbow_link": [1.0, 0.0, 0.25, 0.0],
                 "right_shoulder_pitch_link": [1.0, -0.25, 0.1, 0.0], "left_elbow_link": [1.0, 0.0, 0.25, 0.0]}


class UnitreeH1(BaseRobotHumanoid):
    """Unitree H1 (unitreeH1.py). Default: arms fixed in a reoriented pose, back joint active: 17 dofs, 11 motors."""
    valid_task_confs = ValidTaskConf(tasks=["walk", "run", "carry"], data_types=["real", "perfect"])
    _xml_rel = ("unitree_h1", "h1.xml")

    def __init__(self, disable_arms=True, disable_back_joint=False, hold_weight=False, weight_mass=None, **kwargs):
        super().__init__(disable_arms=disable_arms, disable_back_joint=disable_back_joint, hold_weight=hold_weight,
                         weight_mass=weight_mass, **kwargs)

    def _collision_groups_spec(self):
        return [("floor", ["floor"]), ("foot_r", ["right_foot"]), ("foot_l", ["left_foot"])]

    @staticmethod
    def _get_grf_size():
        return 6

    def _grf_group_names(self):
        return ["foot_r", "foot_l"]

    def _add_weight(self, h, mass):        # unitreeH1.py:425-444 (the arms keep their default pose)
        w = h.add(h.find("body", "torso_link"), "body", name="weight")
        h.add(w, "geom", type="box", size="0.1 0.18 0.1", pos="0.35 0 0.1", group="0", mass=repr(float(mass)))
        return h

    def _modify_xml(self, xml_handle):
        if self._disable_arms:
            for name, quat in _H1_ARM_QUATS.items():       # unitreeH1.py:447-468
                xml_handle.find("body", name).set("quat", " ".join(repr(float(x)) for x in quat))
        return xml_handle

    def _get_xml_modifications(self):
        joints, motors = [], []
        if self._disable_arms:
            joints += _H1_ARMS
            motors += [j + "_actuator" for j in _H1_ARMS]
        if self._disable_back_joint:
            joints += ["back_bkz"]
            motors += ["back_bkz_actuator"]
        return joints, motors, []

    def _has_fallen_terms(self):
        # unitreeH1.py:362-370: the rotation window is +-pi/8 (Atlas/Talos use +-pi/10)
        return [("q_pelvis_ty", -0.3, 0.1), ("q_pelvis_tilt", -np.pi / 4.5, np.pi / 12),
                ("q_pelvis_list", -np.pi / 12, np.pi / 8), ("q_pelvis_rotation", -np.pi / 8, np.pi / 8)]

    @staticmethod
    def _get_observation_specification():
        joints = _PELVIS + ["back_bkz"] + _H1_ARMS + _LEGS
        return [("q_" + j, j, ObservationType.JOINT_POS) for j in joints] + \
               [("dq_" + j, j, ObservationType.JOINT_VEL) for j in joints]

    @staticmethod
    def _get_action_specification():
        return ["back_bkz_actuator"] + [j + "_actuator" for j in _H1_ARMS] + [j + "_actuator" for j in _LEGS]

    @staticmethod
    def generate(task="walk", dataset_type="real", **kwargs):
        stub = "05-run_UnitreeH1.npz" if task == "run" else "02-constspeed_UnitreeH1.npz"
        return UnitreeH1._generate(stub, task, dataset_type, clip_trajectory_to_joint_ranges=True, **kwargs)


_G1_ARMS = ["%s_%s_joint" % (side, j) for side in ("right", "left")
            for j in ("shoulder_pitch", "shoulder_roll", "shoulder_yaw", "elbow_pitch", "elbow_roll")]
_G1_JOINTS = _PELVIS + ["%s_%s_joint" % (side, j) for side in ("left", "right")
                        for j in ("hip_pitch", "hip_roll", "hip_yaw", "knee", "ankle_pitch", "ankle_roll")] + \
    ["torso_joint"] + ["%s_%s_joint" % (side, j) for side in ("left", "right")
                       for j in ("shoulder_pitch", "shoulder_roll", "shoulder_yaw", "elbow_pitch", "elbow_roll")]
_G1_ARM_QUATS = {"left_shoulder_pitch_link": [1.0, 0.25, 0.1, 0.0], "right_elbow_pitch_link": [1.0, 0.0, 0.25, 0.0],
                 "right_shoulder_pitch_link": [1.0, -0.25, 0.1, 0.0], "left_elbow_pitch_link": [1.0, 0.0, 0.25, 0.0]}


class UnitreeG1(BaseRobotHumanoid):
    """Unitree G1 (unitreeG1.py): 29 dofs / 23 motors with arms (default). Observation and action order follow the
    joints / motors of g1.xml (unitreeG1.py:450-481); the feet touch the floor through four small spheres each."""
    valid_task_confs = ValidTaskConf(tasks=["walk", "run"], data_types=["real", "perfect"])
    _xml_rel = ("unitree_g1", "g1.xml")

    def __init__(self, disable_arms=False, disable_back_joint=False, **kwargs):
        super().__init__(disable_arms=disable_arms, disable_back_joint=disable_back_joint, hold_weight=False, **kwargs)

    def _collision_groups_spec(self):       # unitreeG1.py:263-271
        return [("floor", ["floor"])] + [("%s_foot_%d" % (s, k), ["%s_foot_%d_col" % (s, k)])
                                         for s in ("right", "left") for k in (1, 2, 3, 4)]

    @staticmethod
    def _get_grf_size():
        return 24

    def _grf_group_names(self):              # unitreeG1.py:295-317
        return ["%s_foot_%d" % (s, k) for s in ("right", "left") for k in (1, 2, 3, 4)]

    def _modify_xml(self, xml_handle):
        if self._disable_arms:
            for name, quat in _G1_ARM_QUATS.items():       # unitreeG1.py:426-448
                xml_handle.find("body", name).set("quat", " ".join(repr(float(x)) for x in quat))
        return xml_handle

    def _get_xml_modifications(self):
        joints, motors = [], []
        if self._disable_arms:
            joints += _G1_ARMS
            motors += _G1_ARMS                      # the motors carry the joints' names
        if self._disable_back_joint:
            joints += ["torso_joint"]
            motors += ["torso_joint"]
        return joints, motors, []

    def _has_fallen_terms(self):                     # unitreeG1.py:372-376
        return [("q_pelvis_ty", -0.3, 0.1), ("q_pelvis_tilt", -np.pi / 4.5, np.pi / 12),
                ("q_pelvis_list", -np.pi / 12, np.pi / 8), ("q_pelvis_rotation", -np.pi / 8, np.pi / 8)]

    @staticmethod
    def _get_observation_specification():
        return [("q_" + j, j, ObservationType.JOINT_POS) for j in _G1_JOINTS] + \
               [("dq_" + j, j, ObservationType.JOINT_VEL) for j in _G1_JOINTS]

    @staticmethod
    def _get_action_specification():
        return list(_G1_JOINTS[6:])

    @staticmethod
    def generate(task="walk", dataset_type="real", **kwargs):
        stub = "05-run_UnitreeG1.npz" if task == "run" else "02-constspeed_UnitreeG1.npz"
        return UnitreeG1._generate(stub, task, dataset_type, clip_trajectory_to_joint_ranges=True, **kwargs)
