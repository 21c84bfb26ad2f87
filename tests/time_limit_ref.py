"""Reference model of the time limit (include/locosim.h locosim_set_time_limit / locosim_get_episode_stats) for the tests:
the header's semantics restated in Python around one env of the fp64 oracle (oracle_binding.OracleEnv). The oracle supplies
the physics, the reward, the absorbing flag and, under the tracking reward, the trajectory cursor; everything the time limit
adds is integer bookkeeping and lives here. Written from the header, not from the kernels. TEST INFRASTRUCTURE ONLY."""
import ctypes

from loco_mujoco_b200.task import REWARD_TRACKING


def oracle_cursor(oe):
    """trajectory cursor (traj * traj_len + sample) the oracle env keeps for its tracking reward"""
    oe.lib.refenv_cursor.restype = ctypes.c_int
    oe.lib.refenv_cursor.argtypes = [ctypes.c_void_p]
    return int(oe.lib.refenv_cursor(oe.h))


class TimeLimitRef:
    """One oracle env with a time limit. No auto-reset: the caller resets, and until then a finished env stays finished
    (the engine with auto_reset = 0)."""

    def __init__(self, oe, env):
        self.oe = oe
        self.traj_len = env.trajectories.trajectory_length
        self.tracking = env.task_spec().reward_type == REWARD_TRACKING
        self.max_episode_steps, self.end_of_trajectory = 0, False
        self._cursor = 0
        self.length, self.ret, self.last_length, self.last_ret = 0, 0.0, 0, 0.0

    def set_time_limit(self, max_episode_steps=0, end_of_trajectory=False):
        assert max_episode_steps >= 0
        self.max_episode_steps, self.end_of_trajectory = int(max_episode_steps), bool(end_of_trajectory)

    def reset_to(self, traj_no, step_no):
        """a reset of any kind restarts the running length and return and keeps the last finished episode's"""
        self._cursor = int(traj_no) * self.traj_len + int(step_no)
        self.length, self.ret = 0, 0.0
        return self.oe.reset_to(traj_no, step_no)

    def cursor(self):
        # under the tracking reward the oracle's step advances (and clamps) the cursor itself: one advance per step
        return oracle_cursor(self.oe) if self.tracking else self._cursor

    def step_ex(self, action):
        """-> (obs, reward, absorbing, truncated); absorbing wins"""
        obs, r, absorbing = self.oe.step(action)
        self.length += 1
        self.ret += r                                   # (fp64, in step order; the engine sums in fp32)
        truncated = self.max_episode_steps > 0 and self.length >= self.max_episode_steps
        if self.end_of_trajectory:
            if not self.tracking and self._cursor % self.traj_len + 1 < self.traj_len:
                self._cursor += 1
            truncated = truncated or self.cursor() % self.traj_len == self.traj_len - 1
        truncated = truncated and not absorbing
        if absorbing or truncated:
            self.last_length, self.last_ret = self.length, self.ret
        return obs, r, absorbing, truncated

    def episode_stats(self):
        return self.length, self.ret, self.last_length, self.last_ret

    def close(self):
        self.oe.close()
