"""
HumanoidTorque (tasks walk / run, real dataset) on the batched CUDA engine.
Mirrors /root/reference/loco_mujoco/environments/humanoids/base_humanoid.py:12-496 (XML surgery: joint / motor /
equality removal :86-127, box feet :435-472, arm re-orientation :474-496; observation/action specification :292-433;
_has_fallen :129-180; generate :211-290) and humanoids.py:7-317 (HumanoidTorque).
"""
import os
import warnings

import numpy as np

from .. import mjcf
from ..utils.checks import check_validity_task_mode_dataset
from .base import LocoEnv, ObservationType, ValidTaskConf, reference_data_root, ASSET_DIR

_ROOT = ["pelvis_tx", "pelvis_tz", "pelvis_ty", "pelvis_tilt", "pelvis_list", "pelvis_rotation"]
_LEG = ["hip_flexion", "hip_adduction", "hip_rotation", "knee_angle", "ankle_angle", "subtalar_angle", "mtp_angle"]
_LUMBAR = ["lumbar_extension", "lumbar_bending", "lumbar_rotation"]
_ARM = ["arm_flex", "arm_add", "arm_rot", "elbow_flex", "pro_sup", "wrist_flex", "wrist_dev"]
_ARM_MOT = ["shoulder_flex", "shoulder_add", "shoulder_rot", "elbow_flex", "pro_sup", "wrist_flex", "wrist_dev"]


class BaseHumanoid(LocoEnv):
    def _collision_groups_spec(self):
        if self._use_box_feet:      # base_humanoid.py:106-114
            return [("floor", ["floor"]), ("foot_r", ["foot_box_r"]), ("foot_l", ["foot_box_l"])]
        return [("floor", ["floor"]), ("foot_r", ["r_foot"]), ("front_foot_r", ["r_bofoot"]), ("foot_l", ["l_foot"]),
                ("front_foot_l", ["l_bofoot"])]

    def _get_grf_size(self):        # base_humanoid.py:182-191
        return 6 if self._use_box_feet else 12

    def _grf_group_names(self):     # base_humanoid.py:193-209
        return ["foot_r", "foot_l"] if self._use_box_feet else ["foot_r", "front_foot_r", "foot_l", "front_foot_l"]

    def __init__(self, use_muscles=False, use_box_feet=True, disable_arms=True, alpha_box_feet=0.5, _scaling=None,
                 **kwargs):
        if use_muscles:
            raise NotImplementedError("muscle actuation (tendons / <muscle>) is out of scope")
        self._use_muscles, self._use_box_feet, self._disable_arms = use_muscles, use_box_feet, disable_arms
        action_spec = self._get_action_specification(use_muscles)
        observation_spec = self._get_observation_specification()
        joints_to_remove, motors_to_remove, equ = self._get_xml_modifications()
        hide = ["q_" + j for j in joints_to_remove] + ["dq_" + j for j in joints_to_remove]
        observation_spec = [e for e in observation_spec if e[0] not in hide]
        action_spec = [a for a in action_spec if a not in motors_to_remove]
        if kwargs.get("compiled_model") is None:
            root = reference_data_root()
            if root is None:
                raise FileNotFoundError("loco_mujoco model data not found (set LOCO_MUJOCO_PATH)")
            h = mjcf.XmlHandle(os.path.join(root, "environments", "data", "humanoid", "humanoid_torque.xml"))
            if _scaling is not None:
                h = self.scale_body(h, _scaling)
            if use_box_feet or disable_arms:
                h = self._delete_from_xml_handle(h, joints_to_remove, motors_to_remove, equ)
                if use_box_feet:
                    h = self._add_box_feet_to_xml_handle(h, alpha_box_feet, 1.0 if _scaling is None else _scaling)
                if disable_arms:
                    h = self._reorient_arms(h)
        else:
            h = None
        super().__init__(h, action_spec, observation_spec, self._collision_groups_spec(), **kwargs)

    def create_dataset(self, ignore_keys=None):
        if ignore_keys is None:
            ignore_keys = ["q_pelvis_tx", "q_pelvis_tz"]
        return super().create_dataset(ignore_keys)

    def _get_xml_modifications(self):
        joints, motors, equ = [], [], []
        if self._use_box_feet:
            joints += ["subtalar_angle_l", "mtp_angle_l", "subtalar_angle_r", "mtp_angle_r"]
            motors += ["mot_" + j for j in joints]
            equ += [j + "_constraint" for j in joints]
        if self._disable_arms:
            arms = ["%s_%s" % (j, s) for s in ("r", "l") for j in _ARM]
            joints += arms
            motors += ["mot_%s_%s" % (j, s) for s in ("r", "l") for j in _ARM_MOT]
            equ += ["wrist_flex_r_constraint", "wrist_dev_r_constraint", "wrist_flex_l_constraint",
                    "wrist_dev_l_constraint"]
        return joints, motors, equ

    def _has_fallen_terms(self):
        return [("q_pelvis_ty", -0.46, 0.1), ("q_pelvis_tilt", -np.pi / 4.5, np.pi / 12),
                ("q_pelvis_list", -np.pi / 12, np.pi / 8), ("q_pelvis_rotation", -np.pi / 9, np.pi / 9),
                ("q_lumbar_extension", -np.pi / 4, np.pi / 10), ("q_lumbar_bending", -np.pi / 10, np.pi / 10),
                ("q_lumbar_rotation", -np.pi / 4.5, np.pi / 4.5)]

    @staticmethod
    def _add_box_feet_to_xml_handle(h, alpha_box_feet, scaling=1.0):
        size = (np.array([0.112, 0.03, 0.05]) * scaling).tolist()
        pos = (np.array([-0.09, 0.019, 0.0]) * scaling).tolist()
        h.add(h.find("body", "toes_l"), "geom", name="foot_box_l", type="box", size=size, pos=pos, euler=[0.0, 0.15, 0.0])
        h.add(h.find("body", "toes_r"), "geom", name="foot_box_r", type="box", size=size, pos=pos, euler=[0.0, -0.15, 0.0])
        for g in ("r_foot", "r_bofoot", "l_foot", "l_bofoot"):
            e = h.find("geom", g)
            e.set("contype", "0")
            e.set("conaffinity", "0")
        return h

    @staticmethod
    def _reorient_arms(h):
        for name, quat in (("humerus_l", [1.0, -0.1, -1.0, -0.1]), ("ulna_l", [1.0, 0.6, 0.0, 0.0]),
                           ("humerus_r", [1.0, 0.1, 1.0, -0.1]), ("ulna_r", [1.0, -0.6, 0.0, 0.0])):
            h.find("body", name).set("quat", " ".join(repr(x) for x in quat))
        return h

    @staticmethod
    def _get_observation_specification():
        joints = _ROOT + ["%s_r" % j for j in _LEG] + ["%s_l" % j for j in _LEG] + _LUMBAR + \
                 ["%s_r" % j for j in _ARM] + ["%s_l" % j for j in _ARM]
        return [("q_" + j, j, ObservationType.JOINT_POS) for j in joints] + \
               [("dq_" + j, j, ObservationType.JOINT_VEL) for j in joints]

    @staticmethod
    def _get_action_specification(use_muscles=False):
        return ["mot_lumbar_ext", "mot_lumbar_bend", "mot_lumbar_rot"] + \
               ["mot_%s_%s" % (j, s) for s in ("r", "l") for j in _ARM_MOT] + \
               ["mot_%s_%s" % (j, s) for s in ("r", "l") for j in _LEG]

    @classmethod
    def _generate(cls, stubs, task="walk", dataset_type="real", debug=False, **kwargs):
        check_validity_task_mode_dataset(cls.__name__, task, None, dataset_type, *cls.valid_task_confs.get_all())
        if dataset_type != "real":
            raise NotImplementedError("perfect datasets are not shipped (network download in the reference)")
        reward_type = kwargs.pop("reward_type", "target_velocity")
        reward_params = kwargs.pop("reward_params", dict(target_velocity=1.25 if task == "walk" else 2.5))
        root = reference_data_root()
        if root is not None:
            mdp = cls(reward_type=reward_type, reward_params=reward_params, **kwargs)
            path = os.path.join(root, "datasets", "humanoids", "real", stubs[task])
            if debug or not os.path.exists(path):
                if not os.path.exists(path) and not debug:
                    warnings.warn("Datasets not found, falling back to test datasets. Please download and install "
                                  "the datasets to use this environment for imitation learning!")
                path = os.path.join(root, "datasets", "humanoids", "real", "mini_datasets", stubs[task])
            mdp.load_trajectory(dict(traj_path=path, traj_dt=1 / 500.0, control_dt=mdp.dt))
        else:
            from .. import modelpack
            asset = np.load(os.path.join(ASSET_DIR, "%s.%s.npz" % (cls.__name__, task)), allow_pickle=False)
            model = modelpack.from_npz_dict({k[6:]: asset[k] for k in asset.files if k.startswith("model_")})
            mdp = cls(reward_type=reward_type, reward_params=reward_params, compiled_model=model, **kwargs)
            mdp.load_trajectory(dict(processed={k[5:]: asset[k] for k in asset.files if k.startswith("traj_")}))
        return mdp


class HumanoidTorque(BaseHumanoid):
    valid_task_confs = ValidTaskConf(tasks=["walk", "run"], data_types=["real", "perfect"])

    def __init__(self, **kwargs):
        if "use_muscles" in kwargs:
            assert kwargs.pop("use_muscles") is False, "Activating muscles in this environment not allowed. "
        super().__init__(use_muscles=False, **kwargs)

    @staticmethod
    def generate(task="walk", dataset_type="real", **kwargs):
        return HumanoidTorque._generate({"walk": "02-constspeed_reduced_humanoid.npz",
                                         "run": "05-run_reduced_humanoid.npz"}, task, dataset_type, **kwargs)


class HumanoidTorque4Ages(BaseHumanoid):
    """HumanoidTorque scaled to one of four body sizes (base_humanoid_4_ages.py:28-105,243-277,305-358): 0.4 (infant),
    0.6, 0.8, 1.0 (adult); the 2-bit env id is appended to the observation and scales the default reward's target.

    Modes "1".."4" (one scaling) are this class. Mode "all" mixes four models of DIFFERENT kinematics (body offsets, mesh and
    foot sizes, gears) in one env; the engine's multi-model mechanism only swaps inertial / joint parameters, so mode "all"
    is a composite of four single-scaling envs, one engine each: `HumanoidTorque4AgesAll` below."""
    valid_task_confs = ValidTaskConf(tasks=["walk", "run"], modes=["all", "1", "2", "3", "4"], data_types=["real", "perfect"])
    _default_scalings = [0.4, 0.6, 0.8, 1.0]
    _hidable_obs = ("positions", "velocities", "foot_forces", "env_type")

    def _user_feature_name(self):
        return "env_type"

    def __init__(self, scaling=None, scaling_trajectory_map=None, **kwargs):
        if "use_muscles" in kwargs:
            assert kwargs.pop("use_muscles") is False, "Activating muscles in this environment not allowed. "
        scalings = self._default_scalings if scaling is None else (scaling if type(scaling) == list else [scaling])
        if len(scalings) != 1:
            raise NotImplementedError("HumanoidTorque4Ages with several scalings in one env (mode 'all'): the models differ "
                                      "in kinematics; create one env per scaling")
        self._scalings = scalings
        target = kwargs.get("reward_params")
        if kwargs.get("reward_type") == "multi_target_velocity":
            # MultiTargetVelocityReward (utils/reward.py:77-97): target = target_velocity * scaling of the env id
            kwargs["reward_type"] = "target_velocity"
            kwargs["reward_params"] = dict(target_velocity=target["target_velocity"] * scalings[0])
        super().__init__(use_muscles=False, _scaling=scalings[0], **kwargs)
        idx = self._default_scalings.index(scalings[0]) if scalings[0] in self._default_scalings else 0
        self._model_user_features = [(float((idx >> 1) & 1), float(idx & 1))]      # mushroom _get_env_id_map: binary id

    def _get_observation_space(self):
        lo, hi = super()._get_observation_space()
        return np.concatenate([lo, np.zeros(2)]), np.concatenate([hi, np.ones(2)])

    @staticmethod
    def scale_body(h, scaling):
        head_geoms = ["hat_skull", "hat_jaw", "hat_ribs_cap"]
        for mesh in h.root.iter("mesh"):
            if mesh.get("name") not in head_geoms and mesh.get("file") is not None:
                sc = np.array([float(x) for x in mesh.get("scale", "1 1 1").split()]) * scaling
                mesh.set("scale", " ".join(repr(float(x)) for x in sc))
        wb = h.root.find("worldbody")
        for g in wb.iter("geom"):
            if g.get("name") in head_geoms:
                g.set("pos", "0.0 %r 0.0" % (-0.5 * (1 - scaling)))
        for b in wb.iter("body"):
            pos = np.array([float(x) for x in b.get("pos", "0 0 0").split()]) * scaling
            b.set("pos", " ".join(repr(float(x)) for x in pos))
            inertial = b.find("inertial")
            inertial.set("mass", repr(float(inertial.get("mass")) * scaling ** 3))
            fi = np.array([float(x) for x in inertial.get("fullinertia").split()])
            assert np.array_equal(fi[3:], np.zeros(3))
            inertial.set("fullinertia", " ".join(repr(float(x)) for x in fi * scaling ** 5))
        for a in h.root.find("actuator"):
            gear = np.array([float(x) for x in a.get("gear", "1").split()]) * scaling ** 2
            a.set("gear", " ".join(repr(float(x)) for x in gear))
        return h

    @classmethod
    def _generate4(cls, task="walk", mode="all", dataset_type="real", debug=False, **kwargs):
        check_validity_task_mode_dataset(cls.__name__, task, mode, dataset_type, *cls.valid_task_confs.get_all())
        if dataset_type != "real":
            raise NotImplementedError("perfect datasets are not shipped (network download in the reference)")
        if mode == "all":
            return HumanoidTorque4AgesAll(task, dataset_type=dataset_type, debug=debug, **kwargs)
        scaling = cls._default_scalings[int(mode) - 1]
        reward_type = kwargs.pop("reward_type", "multi_target_velocity")
        reward_params = kwargs.pop("reward_params", dict(target_velocity=1.25 if task == "walk" else 2.5))
        stub = ("02-constspeed" if task == "walk" else "05-run") + "_reduced_humanoid_POMDP_%s.npz" % mode
        root = reference_data_root()
        if root is not None:
            mdp = cls(scaling=scaling, reward_type=reward_type, reward_params=reward_params, **kwargs)
            path = os.path.join(root, "datasets", "humanoids", "real", stub)
            if debug or not os.path.exists(path):
                path = os.path.join(root, "datasets", "humanoids", "real", "mini_datasets", stub)
            mdp.load_trajectory(dict(traj_path=path, traj_dt=1 / 500.0, control_dt=mdp.dt))
        else:
            from .. import modelpack
            asset = np.load(os.path.join(ASSET_DIR, "%s.%s.%s.npz" % (cls.__name__, task, mode)), allow_pickle=False)
            model = modelpack.from_npz_dict({k[6:]: asset[k] for k in asset.files if k.startswith("model_")})
            mdp = cls(scaling=scaling, reward_type=reward_type, reward_params=reward_params, compiled_model=model, **kwargs)
            mdp.load_trajectory(dict(processed={k[5:]: asset[k] for k in asset.files if k.startswith("traj_")}))
        return mdp

    @staticmethod
    def generate(task="walk", mode="all", dataset_type="real", **kwargs):
        return HumanoidTorque4Ages._generate4(task, mode, dataset_type, **kwargs)


def _unavailable(feature):
    """A method (or property getter) of HumanoidTorque4AgesAll that refuses `feature`."""
    def refuse(self, *args, **kwargs):
        raise NotImplementedError("%s are not available for HumanoidTorque4Ages mode 'all': use the single-scaling envs "
                                  "(HumanoidTorque4Ages.<task>.<1-4>)" % feature)
    return refuse


class HumanoidTorque4AgesAll:
    """HumanoidTorque4Ages, mode "all" (base_humanoid_4_ages.py:28-105,107-150; humanoids.py:855-892): at the beginning of each
    episode one of the four humanoids (scalings 0.4 / 0.6 / 0.8 / 1.0) is drawn, then a start state from THAT humanoid's
    trajectories. The four models differ in kinematics, so this is a composite of the four single-scaling envs (one engine
    each); the trajectories of `..._POMDP_all.npz` are the four single-scaling datasets in scaling order (default
    `scaling_trajectory_map`), which is what the sub-envs load.

    Drop-in single env (num_envs omitted): the reference's semantics and legacy numpy RNG draw order - model
    (base.py:187-191), trajectory within the model's range (base_humanoid_4_ages.py:132-136), sample (trajectory.py:253-259);
    reproduces the reference goldens HumanoidTorque4Ages.{walk,run}.all.
    Batched (num_envs=N): env i permanently belongs to humanoid i % 4 (the reference redraws the humanoid per episode; a fixed
    assignment keeps the same marginal mix and lets every engine stay homogeneous); everything else as in LocoEnv."""

    def __init__(self, task="walk", dataset_type="real", debug=False, num_envs=None, env_id_offset=0, **kwargs):
        n = None if num_envs is None else int(num_envs)
        self.num_envs = 1 if n is None else n
        self.batched = n is not None
        self._index = None
        self.subs = []
        off = int(env_id_offset)
        for k in range(4):
            kw = dict(kwargs)
            if self.batched:
                nk = len(range(k, n, 4))
                if nk == 0:
                    raise ValueError("mode 'all' needs num_envs >= 4 (one env per humanoid)")
                kw.update(num_envs=nk, env_id_offset=off)
                off += nk
            self.subs.append(HumanoidTorque4Ages._generate4(task, str(k + 1), dataset_type, debug=debug, **kw))
        self._current_model_idx = 0
        self.info = self.subs[0].info
        self.trajectories = None            # per humanoid: self.subs[k].trajectories

    # ---- everything that does not depend on the humanoid comes from the first sub-env ----
    def __getattr__(self, name):
        if name in ("subs", "__setstate__"):
            raise AttributeError(name)
        return getattr(self.subs[0], name)

    @property
    def dt(self):
        return self.subs[0].dt

    # ---- the per-env outputs and the dynamics queries: the four humanoids differ in their bodies and the envs are
    # interleaved over four engines ----
    body_index = _unavailable("applied forces (xfrc_applied / qfrc_applied / body_index)")
    xfrc_applied = qfrc_applied = property(body_index)
    body_state = next_body_state = property(_unavailable("body outputs (body_state / next_body_state)"))
    contact_wrench = property(_unavailable("contact outputs (contact_wrench)"))
    dof_outputs = property(_unavailable("dof outputs (dof_outputs)"))
    geom_index = _unavailable("contact lists (contacts / geom_index / geom_names)")
    contacts = geom_names = property(geom_index)
    create_dataset_bodies = _unavailable("reference outputs (reference_body_state / next_reference_body_state / "
                                         "create_dataset_bodies)")
    reference_body_state = next_reference_body_state = property(create_dataset_bodies)
    inverse_dynamics = create_dataset_inverse = dof_index = _unavailable(
        "inverse dynamics (inverse_dynamics / create_dataset_inverse / dof_index)")
    dynamics_terms = _unavailable("the dynamics terms (dynamics_terms)")
    forward_dynamics = _unavailable("the forward dynamics (forward_dynamics)")
    save_state = _unavailable("saved states (save_state)")
    load_state = _unavailable("saved states (load_state)")
    ray_cast = camera = render = _unavailable("ray casting (ray_cast / camera / render)")

    def _scatter(self, parts):
        """Per-humanoid tensors [n_k, ...] -> one tensor in env order (env i = humanoid i % 4, its (i // 4)-th env)."""
        import torch
        if self._index is None:
            order = [i for k in range(4) for i in range(k, self.num_envs, 4)]          # env ids in concatenation order
            inv = torch.empty(self.num_envs, dtype=torch.long)
            inv[torch.tensor(order)] = torch.arange(self.num_envs)
            self._index = inv.to(parts[0].device)
        return torch.cat(parts, dim=0)[self._index]

    def reset(self, obs=None):
        if obs is not None:
            raise TypeError("Initializing the environment from an observation is not allowed in this environment.")
        if not self.batched:
            import torch
            model_no = np.random.randint(0, 4)                                      # base.py:187-191
            self._current_model_idx = model_no
            sub = self.subs[model_no]
            sub._reward_function.reset_state()
            np.random.randint(model_no, model_no + 1)                               # traj_no within the model's range (one trajectory each)
            sub.trajectories.reset_trajectory(traj_no=0)                           # draws the sample
            eng = sub._get_engine()
            out = eng.reset(traj_no=torch.zeros(1, dtype=torch.int32, device=eng.device),
                            step_no=torch.tensor([sub.trajectories.subtraj_step_no], dtype=torch.int32, device=eng.device))
            sub._obs = out[0].double().cpu().numpy()
            return sub._obs.copy()
        return self._scatter([s.reset() for s in self.subs])

    def step(self, action):
        if not self.batched:
            return self.subs[self._current_model_idx].step(action)
        outs = [s.step(action[k::4].contiguous()) for k, s in enumerate(self.subs)]
        obs, rew, done = (self._scatter([o[j] for o in outs]) for j in range(3))
        # (every info entry is a per-env tensor: next_obs, and with a time limit truncated / episode_length / episode_return)
        return obs, rew, done, {k: self._scatter([o[3][k] for o in outs]) for k in outs[0][3]}

    def create_dataset(self, ignore_keys=None):
        """The four humanoids' datasets, concatenated in scaling order (the layout of the reference's `_all` dataset)."""
        parts = [s.create_dataset(ignore_keys=ignore_keys) for s in self.subs]
        return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}

    def stop(self):
        pass
