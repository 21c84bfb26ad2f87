"""
Gymnasium interface (reference: /root/reference/loco_mujoco/environments/gymnasium.py:11-173).
`gymnasium` itself is optional: when it is importable the wrapper subclasses gymnasium.Env and is registered as
"LocoMujoco" (reference registration: environments/humanoids/__init__.py:20-25); otherwise the same class works
stand-alone through `loco_mujoco_b200.make_gym("LocoMujoco", env_name=...)`.
"""
import numpy as np

from .base import LocoEnv

try:                                    # pragma: no cover - depends on the host environment
    import gymnasium as _gym
    from gymnasium import spaces as _spaces
    _Base = _gym.Env
except Exception:                       # gymnasium is not installed in the build image
    _gym = None
    _Base = object

    class _BoxSpace:
        def __init__(self, low, high, shape, dtype):
            self.low = np.full(shape, low, dtype=dtype)
            self.high = np.full(shape, high, dtype=dtype)
            self.shape, self.dtype = tuple(shape), dtype

        def sample(self):
            lo = np.where(np.isfinite(self.low), self.low, -1.0)
            hi = np.where(np.isfinite(self.high), self.high, 1.0)
            return np.random.uniform(lo, hi).astype(self.dtype)

    class _spaces:
        Box = _BoxSpace


class GymnasiumWrapper(_Base):
    """step -> (obs, reward, terminated, truncated, info); reset(seed, options) -> (obs, {}). `truncated` is False unless the
    env was made with `time_limit` / `truncate_at_trajectory_end` (LocoEnv); the caller resets a truncated env."""

    metadata = {"render_modes": ["human", "rgb_array"], "render_fps": 100}

    def __init__(self, env_name, render_mode=None, **kwargs):
        self.spec = None
        self._env = LocoEnv.make(env_name, **kwargs)
        self.render_mode = render_mode
        self.metadata = dict(self.metadata, render_fps=1.0 / self._env.dt)
        self.observation_space = self._convert_space(self._env.info.observation_space)
        self.action_space = self._convert_space(self._env.info.action_space)

    def step(self, action):
        obs, reward, absorbing, info = self._env.step(action)
        return obs, reward, absorbing, info.get("truncated", False), info

    def reset(self, *, seed=None, options=None):
        if seed is not None and _gym is not None:
            super().reset(seed=seed)
        return self._env.reset(), {}

    def render(self):
        """render_mode "rgb_array": the env's frame as uint8 [height, width, 3] (the reference's swap of render(True)'s
        [width, height, 3]). "human" needs a window, which this headless engine does not have."""
        if self.render_mode == "rgb_array":
            return np.swapaxes(self._env.render(True), 0, 1)
        if self.render_mode == "human":
            raise NotImplementedError("render_mode 'human' needs a viewer window: the engine is headless, use 'rgb_array'")
        return None

    def close(self):
        self._env.stop()

    def create_dataset(self, **kwargs):
        return self._env.create_dataset(**kwargs)

    def play_trajectory(self, **kwargs):
        return self._env.play_trajectory(**kwargs)

    @property
    def unwrapped(self):
        return self._env

    @staticmethod
    def _convert_space(space):
        low, high = np.min(space.low), np.max(space.high)
        return _spaces.Box(low, high, shape=space.shape, dtype=np.float64) if _gym is None else \
            _spaces.Box(low, high, space.shape, np.float64)


class VectorGymnasiumWrapper:
    """Batched counterpart with the Gymnasium VectorEnv call contract (SURVEY 8(f).4): `num_envs` independent copies on
    one GPU, autoreset in the same step ("SAME_STEP" mode: for sub-envs that terminated, `obs` is already the first
    observation of the next episode and `info["final_obs"]` holds the terminal observation of ALL sub-envs, to be
    masked with `terminated | truncated`). `time_limit` / `truncate_at_trajectory_end` (LocoEnv keyword arguments) turn the
    time limit on: `truncated` is then the engine's flag, and `info["episode"] = {"r": return, "l": length}` with the mask
    `info["_episode"]` reports the episodes that ended in this step (the keys of Gymnasium's RecordEpisodeStatistics).
    Tensors stay on the device (torch.cuda) unless `to_numpy=True`.
    The reference has no vector interface; its single-env wrapper is `GymnasiumWrapper` (gymnasium.py:11-173)."""

    def __init__(self, env_name, num_envs, device="cuda:0", seed=0, to_numpy=False, time_limit=None,
                 truncate_at_trajectory_end=False, **kwargs):
        self._env = LocoEnv.make(env_name, num_envs=num_envs, device=device, seed=seed, time_limit=time_limit,
                                 truncate_at_trajectory_end=truncate_at_trajectory_end, **kwargs)
        self.num_envs = int(num_envs)
        self._to_numpy = to_numpy
        one_obs, one_act = self._env.info.observation_space, self._env.info.action_space
        self.single_observation_space = GymnasiumWrapper._convert_space(one_obs)
        self.single_action_space = GymnasiumWrapper._convert_space(one_act)
        self.observation_space = _spaces.Box(np.min(one_obs.low), np.max(one_obs.high),
                                             shape=(self.num_envs,) + tuple(one_obs.shape), dtype=np.float64)
        self.action_space = _spaces.Box(np.min(one_act.low), np.max(one_act.high),
                                        shape=(self.num_envs,) + tuple(one_act.shape), dtype=np.float64)
        self.metadata = {"autoreset_mode": "same_step", "render_fps": 1.0 / self._env.dt}

    def _out(self, t):
        return t.detach().cpu().numpy() if self._to_numpy else t

    def reset(self, *, seed=None, options=None):
        return self._out(self._env.reset()), {}

    def step(self, actions):
        import torch
        if not torch.is_tensor(actions):
            actions = torch.as_tensor(np.asarray(actions, dtype=np.float32), device=self._env._get_engine().device)
        obs, reward, done, info = self._env.step(actions)
        out = {"final_obs": self._out(obs)}
        if "truncated" in info:
            truncated = info["truncated"]
            out["episode"] = {"r": self._out(info["episode_return"]), "l": self._out(info["episode_length"])}
            out["_episode"] = self._out(done | truncated)
        else:
            truncated = torch.zeros_like(done)
        return self._out(info["next_obs"]), self._out(reward), self._out(done), self._out(truncated), out

    def close(self):
        self._env.stop()

    @property
    def unwrapped(self):
        return self._env


def make_gym(env_id, **kwargs):
    if env_id != "LocoMujoco":
        raise KeyError(env_id)
    return GymnasiumWrapper(**kwargs)


if _gym is not None:                    # pragma: no cover
    try:
        _gym.register("LocoMujoco", entry_point="loco_mujoco_b200.environments.gymnasium:GymnasiumWrapper")
    except Exception:
        pass
