"""Time limit (include/locosim.h locosim_set_time_limit), CPU tier: the reference model of the header's semantics around the
fp64 oracle (tests/time_limit_ref.py), which the GPU tier compares the engine with, against a recount of the same rollout, and
the host logic of the Python layers without a device (argument validation, the split of the done byte, the info keys).
The GPU tier is tests/test_time_limit_gpu.py."""
import numpy as np
import pytest

from helpers import make_env, oracle_env
from time_limit_ref import TimeLimitRef, oracle_cursor

TASK = "UnitreeA1.simple"


@pytest.fixture()
def a1(oracle, bundled_only):
    env = make_env(TASK)
    oe = TimeLimitRef(oracle_env(oracle, env), env)
    yield env, oe
    oe.close()


def test_oracle_truncates_on_the_step_that_reaches_the_limit(a1):
    env, oe = a1
    oe.set_time_limit(7, 0)
    oe.reset_to(0, 0)
    rewards, flags = [], []
    for k in range(9):                                # (no auto-reset in the oracle: a finished env stays finished)
        _, r, ab, tr = oe.step_ex(np.zeros(12))
        rewards.append(r)
        flags.append((ab, tr))
        if k == 6:
            at_limit = oe.episode_stats()
    assert flags == [(False, False)] * 6 + [(False, True)] * 3
    # length and return against a recount in the same order
    ret = 0.0
    for r in rewards[:7]:
        ret += r
    assert at_limit == (7, ret, 7, ret)
    ln, run, last_ln, last_ret = oe.episode_stats()
    assert (ln, last_ln) == (9, 9) and run == last_ret == sum_in_order(rewards)
    oe.reset_to(0, 3)                                 # a reset restarts the running pair and keeps the finished one
    assert oe.episode_stats() == (0, 0.0, 9, last_ret)
    assert oe.step_ex(np.zeros(12))[2:] == (False, False)


def sum_in_order(xs):
    s = 0.0
    for x in xs:
        s += x
    return s


def test_oracle_limit_off_is_the_oracle_step(oracle, a1):
    env, oe = a1
    other = oracle_env(oracle, env)
    rng = np.random.default_rng(3)
    oe.reset_to(1, 20)
    other.reset_to(1, 20)
    for _ in range(12):
        a = rng.uniform(-1, 1, 12)
        o1, r1, ab1, tr = oe.step_ex(a)
        o2, r2, ab2 = other.step(a)
        assert np.array_equal(o1, o2) and r1 == r2 and ab1 == ab2 and not tr
        assert oe.cursor() == oracle_cursor(other) == 1 * 100 + 20   # (no tracking reward: it rests)
    other.close()


@pytest.mark.parametrize("back,first_truncated", [(3, 2), (2, 1), (1, 1)])
def test_oracle_end_of_trajectory_off_by_one(a1, back, first_truncated):
    """Reset to sample traj_len - back: the step after which the cursor stands on the last sample is truncated (the step for
    which the reference's get_next_sample() would next return None); reset ONTO the last sample: the first step, and the
    cursor does not move."""
    env, oe = a1
    T = env.trajectories.trajectory_length
    oe.set_time_limit(0, 1)
    oe.reset_to(1, T - back)
    cursors, trunc = [], []
    for _ in range(first_truncated + 1):
        _, _, ab, tr = oe.step_ex(np.zeros(12))
        assert not ab
        trunc.append(tr)
        cursors.append(oe.cursor())
    assert trunc == [False] * (first_truncated - 1) + [True, True]
    want = [min(T + T - back + k + 1, 2 * T - 1) for k in range(first_truncated + 1)]
    assert cursors == want                              # one sample per step, never past the trajectory's last sample
    assert oe.episode_stats()[2] == first_truncated + 1  # (rewritten while the env stays finished)


def test_oracle_tracking_reward_advances_once_per_step(oracle, bundled_only):
    """Under the tracking reward the oracle's step has advanced the cursor already: end_of_trajectory must not advance it
    again, and the rewards are those of the plain step."""
    env = make_env(TASK, reward_type="tracking")
    T = env.trajectories.trajectory_length
    oe, other = TimeLimitRef(oracle_env(oracle, env), env), oracle_env(oracle, env)
    oe.set_time_limit(0, 1)
    oe.reset_to(0, T - 4)
    other.reset_to(0, T - 4)
    for k in range(3):
        _, r, ab, tr = oe.step_ex(np.zeros(12))
        _, r2, _ = other.step(np.zeros(12))
        assert r == r2 and not ab
        assert oe.cursor() == T - 4 + k + 1
        assert tr == (k == 2)
    oe.close()
    other.close()


def test_oracle_absorbing_wins_at_the_limit(a1):
    env, oe = a1
    rng = np.random.default_rng(0)
    actions = rng.uniform(-1, 1, (200, 12))
    oe.reset_to(0, 10)
    fall = None
    for k, a in enumerate(actions):
        if oe.step_ex(a)[2]:
            fall = k + 1
            break
    assert fall is not None and fall > 1, "the seeded actions should make the robot fall"
    oe.set_time_limit(fall, 0)
    oe.reset_to(0, 10)
    rewards = []
    for k in range(fall):
        _, r, ab, tr = oe.step_ex(actions[k])
        rewards.append(r)
        assert (ab, tr) == ((True, False) if k == fall - 1 else (False, False)), k
    assert oe.episode_stats()[2:] == (fall, sum_in_order(rewards))
    # one step earlier the limit is reached by a step that does not fall
    oe.set_time_limit(fall - 1, 0)
    oe.reset_to(0, 10)
    for k in range(fall - 1):
        _, _, ab, tr = oe.step_ex(actions[k])
    assert (ab, tr) == (False, True)


# ---------------------------------------------------------------------------------------------------------------------
# host logic without a device
# ---------------------------------------------------------------------------------------------------------------------
def test_time_limit_argument():
    from loco_mujoco_b200.environments.base import resolve_time_limit
    assert resolve_time_limit(None, 1000) == 0
    assert resolve_time_limit("horizon", 1000) == 1000
    assert resolve_time_limit(250, 1000) == 250
    assert resolve_time_limit(250.0, 1000) == 250
    for bad in (-1, 0, 2.5, "episode", True):
        with pytest.raises(ValueError):
            resolve_time_limit(bad, 1000)
    with pytest.raises(ValueError):
        resolve_time_limit("horizon", 0)


def test_env_arguments(bundled_only):
    env = make_env(TASK, num_envs=4)
    assert not env.time_limited and env._max_episode_steps == 0
    env = make_env(TASK, num_envs=4, time_limit="horizon", horizon=300)
    assert env.time_limited and env._max_episode_steps == 300 and not env._truncate_at_trajectory_end
    env = make_env(TASK, num_envs=4, truncate_at_trajectory_end=True)
    assert env.time_limited and env._max_episode_steps == 0
    with pytest.raises(ValueError):
        make_env(TASK, num_envs=4, time_limit=-5)
    # composites hand the setting to every member
    env = make_env("HumanoidTorque4Ages.walk.all", num_envs=8, time_limit=50)
    assert [s._max_episode_steps for s in env.subs] == [50] * 4


def test_split_done():
    import torch
    from loco_mujoco_b200.engine import split_done
    raw = np.array([0, 1, 2, 0, 1], dtype=np.uint8)
    for done in (raw, torch.from_numpy(raw)):
        ab, tr = split_done(done)
        assert ab.tolist() == [False, True, False, False, True] and tr.tolist() == [False, False, True, False, False]
        assert ab.dtype in (np.bool_, torch.bool)


class FakeEngine:
    """What LocoEnv.step uses of CudaEngine, on CPU tensors: every step returns the done bytes it was given."""

    def __init__(self, n, obs_dim, done):
        import torch
        self.torch, self.n_envs, self.obs_dim, self.device = torch, n, obs_dim, torch.device("cpu")
        self.packed_out = torch.zeros((n * (4 * obs_dim + 5),), dtype=torch.uint8)
        self.next_obs = torch.zeros((n, obs_dim))
        self._done = torch.tensor(done, dtype=torch.uint8)
        self.limit = None
        self.stats_calls = 0

    def views_of(self, packed):
        from loco_mujoco_b200.engine import CudaEngine
        return CudaEngine.views_of(self, packed)

    def step(self, action, auto_reset=True, want_next_obs=True, packed=None):
        obs, reward, done = self.views_of(self.packed_out)
        done.copy_(self._done)
        return obs, reward, done, self.next_obs

    def episode_stats(self):
        t = self.torch
        self.stats_calls += 1
        return (t.zeros(self.n_envs, dtype=t.int32), t.zeros(self.n_envs), t.arange(self.n_envs, dtype=t.int32),
                t.arange(self.n_envs, dtype=t.float32))


@pytest.mark.parametrize("copy_outputs", [True, False])
def test_step_info_keys(bundled_only, copy_outputs):
    import torch
    n = 4
    act = torch.zeros((n, 12))
    env = make_env(TASK, num_envs=n, copy_outputs=copy_outputs)
    env._engine = eng = FakeEngine(n, 37, [0, 1, 0, 1])
    _, _, done, info = env.step(act)
    assert sorted(info) == ["next_obs"] and done.dtype == torch.bool and done.tolist() == [False, True, False, True]
    assert eng.stats_calls == 0                         # the path without a limit asks the engine for nothing more

    env = make_env(TASK, num_envs=n, copy_outputs=copy_outputs, time_limit=5)
    env._engine = eng = FakeEngine(n, 37, [0, 1, 2, 0])
    _, _, done, info = env.step(act)
    assert sorted(info) == ["episode_length", "episode_return", "next_obs", "truncated"]
    assert done.dtype == torch.bool and done.tolist() == [False, True, False, False]
    assert info["truncated"].dtype == torch.bool and info["truncated"].tolist() == [False, False, True, False]
    assert info["episode_length"].tolist() == [0, 1, 2, 3] and info["episode_return"].tolist() == [0.0, 1.0, 2.0, 3.0]


def test_single_env_info(bundled_only):
    env = make_env(TASK)
    env._engine = FakeEngine(1, 37, [2])
    env._obs = np.zeros(37)
    _, _, absorbing, info = env.step(np.zeros(12))
    assert absorbing is False and info == {}            # (bit 1 cannot be set without a limit; the key stays out regardless)
    env = make_env(TASK, truncate_at_trajectory_end=True)
    for byte, want in ((2, (False, True)), (1, (True, False)), (0, (False, False))):
        env._engine = FakeEngine(1, 37, [byte])
        env._obs = np.zeros(37)
        _, _, absorbing, info = env.step(np.zeros(12))
        assert (absorbing, info["truncated"]) == want and type(info["truncated"]) is bool


def test_gymnasium_wrappers_report_truncation(bundled_only):
    import torch
    from loco_mujoco_b200 import GymnasiumWrapper, VectorGymnasiumWrapper
    g = GymnasiumWrapper(TASK + ".real", debug=True, time_limit=3)
    g._env._engine = FakeEngine(1, 37, [2])
    g._env._obs = np.zeros(37)
    assert g.step(np.zeros(12))[2:4] == (False, True)
    g = GymnasiumWrapper(TASK + ".real", debug=True)
    g._env._engine = FakeEngine(1, 37, [1])
    g._env._obs = np.zeros(37)
    assert g.step(np.zeros(12))[2:4] == (True, False)

    v = VectorGymnasiumWrapper(TASK + ".real", 4, debug=True, time_limit=3)
    v._env._engine = FakeEngine(4, 37, [0, 1, 2, 0])
    _, _, term, trunc, info = v.step(torch.zeros((4, 12)))
    assert term.tolist() == [False, True, False, False] and trunc.tolist() == [False, False, True, False]
    assert info["_episode"].tolist() == [False, True, True, False]
    assert info["episode"]["l"].tolist() == [0, 1, 2, 3] and info["episode"]["r"].tolist() == [0.0, 1.0, 2.0, 3.0]
    v = VectorGymnasiumWrapper(TASK + ".real", 4, debug=True)
    v._env._engine = FakeEngine(4, 37, [0, 1, 0, 0])
    _, _, term, trunc, info = v.step(torch.zeros((4, 12)))
    assert not trunc.any() and sorted(info) == ["final_obs"]
