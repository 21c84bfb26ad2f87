"""UnitreeA1 under PD position control on the GPU: the batched engine against the fp64 oracle from the engine's own pre-step
states (the method of tests/test_gpu_parity.py), on all three launch paths, with the done flags compared bit for bit; the
three launch paths agree bit for bit; and a full-size batch of 4096 envs steps and its dof outputs match the fp64
reference."""
import numpy as np
import pytest
import torch

import dof_outputs_ref as dor
from helpers import blobs, oracle_step_sensitivity
from position_mode import make_position
from test_dof_outputs import within
from test_dof_outputs_gpu import PATHS, _make

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref():
    return dor.load()


@pytest.mark.parametrize("path", list(PATHS))
def test_position_mode_matches_the_oracle(oracle, bundled_only, path):
    """512 envs reset to known trajectory samples, 8 control steps under random actions (auto_reset=False): for sampled envs
    the oracle, reset to the same sample (its goal) and set to the engine's pre-step state and warm start, gives the engine's
    observation (within 2e-3, the tolerance of test_gpu_parity's first step, or within 10x the oracle's own jump where a
    contact switches within the step), done flag (exactly) and, on the first step, reward (1e-3)"""
    n = 512
    env = _make("UnitreeA1.simple+position", path, num_envs=n, seed=5)
    eng = env._get_engine()
    mb, tb = blobs(env)
    rng = np.random.RandomState(0)
    tr = rng.randint(0, env.trajectories.number_of_trajectories, n).astype(np.int32)
    st = rng.randint(0, env.trajectories.trajectory_length, n).astype(np.int32)
    eng.reset(traj_no=torch.tensor(tr, device=eng.device), step_no=torch.tensor(st, device=eng.device))
    alive = np.ones(n, dtype=bool)
    checked, dones, allowed = 0, 0, 0
    for k in range(8):
        act = rng.uniform(-1, 1, (n, 12)).astype(np.float32)
        q0, v0, w0 = (x.cpu().numpy().astype(np.float64) for x in eng.get_state())
        obs, rew, done, _ = eng.step(torch.tensor(act, device=eng.device), auto_reset=False)
        obs, rew, done = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        for i in range(k, n, 7):
            if not alive[i]:
                continue
            oe = oracle.env(mb, tb)
            oe.reset_to(tr[i], st[i])
            oe.set_state(q0[i], v0[i], w0[i])
            o, r, d = oe.step(act[i].astype(np.float64))
            oe.close()
            if not np.allclose(obs[i], o, rtol=2e-3, atol=2e-3):
                gap = oracle_step_sensitivity(oracle, mb, tb, tr[i], st[i], q0[i], v0[i], act[i], o, eps=1e-5, n_probe=8,
                                              relative=True)
                assert np.abs(obs[i] - o).max() <= 10 * gap + 2e-3, (path, k, i, np.abs(obs[i] - o).max(), gap)
                allowed += 1
                alive[i] = False
                continue
            if k == 0:      # (the reward is that of the observation before the step, which the oracle has from its reset)
                assert abs(rew[i] - r) < 1e-3, (path, k, i, rew[i], r)
            assert bool(done[i] & 1) == d, (path, k, i, done[i], d)
            dones += int(d)
            checked += 1
        alive &= ~done.astype(bool)
    assert checked > 300 and allowed <= checked // 20, (checked, allowed)
    assert dones > 0, "no env fell: the done flags were not exercised"


def test_launch_paths_agree_bit_for_bit(bundled_only):
    n = 512
    envs = [_make("UnitreeA1.simple+position", p, num_envs=n, seed=3) for p in PATHS]
    obs = [e.reset() for e in envs]
    assert all(torch.equal(obs[0], o) for o in obs[1:])
    gen = torch.Generator().manual_seed(2)
    for _ in range(8):
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        outs = [e.step(act) for e in envs]
        for o in outs[1:]:
            for x, y in zip(outs[0][:3], o[:3]):
                assert torch.equal(x, y)
    for e in envs[1:]:
        for x, y in zip(envs[0]._get_engine().get_state(), e._get_engine().get_state()):
            assert torch.equal(x, y)


def test_full_size_batch_steps_and_its_dof_outputs_match_the_reference(ref, bundled_only):
    """LocoEnv.make("UnitreeA1.simple", action_mode="position", num_envs=4096): steps on the device, and the dof outputs of
    sampled envs match the fp64 reference's sub-step mean from the engine's own pre-step states"""
    from loco_mujoco_b200 import LocoEnv
    n = 4096
    env = LocoEnv.make("UnitreeA1.simple.real", action_mode="position", num_envs=n, device="cuda:0", seed=2, debug=True)
    eng = env._get_engine()
    d = env.dof_outputs
    mb, tb = blobs(env)
    env.reset()
    gen = torch.Generator().manual_seed(3)
    checked, allowed = 0, 0
    for k in range(5):
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        q0, v0, w0 = (x.cpu().numpy().astype(np.float64) for x in eng.get_state())
        obs, _, _, _ = env.step(act)
        assert bool(torch.isfinite(obs).all())
        rows, an = d.cpu().numpy(), act.cpu().numpy().astype(np.float64)
        for i in range(k, n, 397):
            oe = ref.env(mb, tb)
            oe.set_state(q0[i], v0[i], w0[i])
            want, _, _ = dor.env_step(ref, oe, an[i])
            oe.close()
            ok, err, tol = within(rows[i], want)
            if not ok:
                gap = dor.sensitivity(ref, mb, tb, q0[i], v0[i], an[i], want, warmstart=w0[i], eps=1e-6, n_probe=8)
                ok, err, tol = within(rows[i], want, gap)
                assert ok, (k, i, err, tol, gap)
                allowed += 1
            checked += 1
    assert allowed <= 2, (allowed, checked)
    # the actuator forces are the position actuators' (clamped to +-33.5 N m on the twelve leg dofs, zero on the root)
    assert float(d[:, :6, 0].abs().max()) == 0.0 and float(d[:, 6:, 0].abs().max()) <= 33.5 * (1 + 1e-6)
