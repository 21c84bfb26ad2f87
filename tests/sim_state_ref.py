"""The engine's counter-based per-env draws (locosim.cu mix64, draw_reset, draw_rot_angle, draw_pool_row) restated in Python,
bit for bit: what reset number `episode` of global env `genv` draws. The saved-state tests use them to predict what a
loaded (forked) env's first reset gives. Test infrastructure only."""
import numpy as np

M64 = (1 << 64) - 1


def mix64(z):
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def _key(genv, episode):
    return mix64(((genv & M64) * 0x100000001B3 + (episode & 0xFFFFFFFF)) & M64)


def draw_reset(seed, genv, episode, n_traj, traj_len):
    """(trajectory, sample) of reset number `episode` of global env `genv`"""
    r = mix64((seed & M64) ^ _key(genv, episode))
    return (r & 0xFFFFFFFF) % n_traj, (r >> 32) % traj_len


def draw_rot_angle(seed, genv, episode):
    """setup_random_rot angle (np.float32) of reset number `episode` of global env `genv`"""
    r = mix64(((seed + 0x2545F4914F6CDD1D) & M64) ^ _key(genv, episode))
    return np.float32(r >> 40) * (np.float32(6.283185307179586) / np.float32(16777216.0))


def draw_pool_row(seed, genv, episode, K):
    """parameter-pool row of reset number `episode` of global env `genv` with a pool of K rows"""
    if K <= 1:
        return 0
    r = mix64(((seed + 0x5DEECE66D) & M64) ^ _key(genv, episode))
    return r % K
