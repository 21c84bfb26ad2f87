"""Applied forces (MuJoCo's xfrc_applied / qfrc_applied, include/locosim.h locosim_set_applied_forces) without a GPU:
the fp64 reference (tests/csrc/applied_forces_ref.c) against finite-difference Jacobians, against an actuator and against
the unextended oracle; the serial build of the CUDA core against that reference; the host-side checks."""

import numpy as np
import pytest

import applied_forces_ref
from full_body import make_variant
from helpers import blobs, make_env

TASKS = ["UnitreeA1.simple", "HumanoidTorque.run", "Atlas.walk+arms"]


@pytest.fixture(scope="module")
def ref():
    return applied_forces_ref.load()


def _pose(env, rng, scale=0.1):
    """a state of the reset table, perturbed (qpos, qvel)"""
    spec = env.task_spec()
    nv = env._model.nv
    table = spec.table.reshape(-1, spec.table.shape[-1])
    row = table[rng.randint(len(table))]
    return row[:nv] + scale * rng.randn(nv), row[nv:2 * nv] + scale * rng.randn(nv)


def _vee(S):
    return np.array([S[2, 1] - S[1, 2], S[0, 2] - S[2, 0], S[1, 0] - S[0, 1]]) * 0.5


@pytest.mark.parametrize("task", TASKS)
def test_wrench_maps_through_the_body_jacobian(ref, bundled_only, task):
    """qfrc_smooth(with the wrench) - qfrc_smooth(without) = Jp^T F + Jr^T tau, with Jp = d xipos / dq and Jr from
    d xmat / dq by central differences of the oracle's own kinematics (nq = nv: slide and hinge joints only)."""
    env = make_variant(task)
    sim = applied_forces_ref.AppliedSim(ref, *blobs(env))
    rng = np.random.RandomState(1)
    nv, nb = sim.nv, sim.nb
    zero_ctrl = np.zeros(env._model.nu)
    worst = 0.0
    for _ in range(3):
        q, v = _pose(env, rng)
        base = sim.forward(q, v, zero_ctrl)
        h = 1e-6
        Jp, Jr = np.zeros((nb, 3, nv)), np.zeros((nb, 3, nv))
        for j in range(nv):
            dq = np.zeros(nv)
            dq[j] = h
            a, b = sim.forward(q + dq, v, zero_ctrl), sim.forward(q - dq, v, zero_ctrl)
            Jp[:, :, j] = (a["xipos"] - b["xipos"]) / (2 * h)
            for k in range(nb):
                Jr[k, :, j] = _vee((a["xmat"][k] - b["xmat"][k]) / (2 * h) @ base["xmat"][k].T)
        for body in rng.choice(np.arange(1, nb), size=min(4, nb - 1), replace=False):
            w = np.zeros((nb, 6))
            w[body] = rng.randn(6) * [40, 40, 40, 5, 5, 5]
            got = sim.forward(q, v, zero_ctrl, xfrc=w)["qfrc_smooth"] - base["qfrc_smooth"]
            want = Jp[body].T @ w[body, :3] + Jr[body].T @ w[body, 3:]
            err = np.abs(got - want).max() / np.abs(want).max()
            worst = max(worst, err)
            assert err < 1e-6, (task, body, err)
        # the world body's row is ignored
        w = np.zeros((nb, 6))
        w[0] = 100.0
        assert np.array_equal(sim.forward(q, v, zero_ctrl, xfrc=w)["qfrc_smooth"], base["qfrc_smooth"])
    sim.close()


def test_qfrc_applied_equals_an_actuator(ref, bundled_only):
    """UnitreeA1's motors (gain 1, no bias, symmetric ctrl ranges): a trajectory under action a and one under action 0 with
    qfrc_applied = gear * gain * ctrl(a) on the actuated dofs agree to fp64 round-off, contacts and all."""
    env = make_env("UnitreeA1.simple")
    m, spec = env._model, env.task_spec()
    assert np.all(np.asarray(m.actuator_bias) == 0) and np.allclose(spec.act_mean, 0)
    gear, gain = np.asarray(m.actuator_gear).ravel(), np.asarray(m.actuator_gain).ravel()
    dof, rng_ = np.asarray(m.actuator_dof), np.asarray(m.actuator_ctrlrange).reshape(-1, 2)
    rng = np.random.RandomState(2)
    a_sim, b_sim = (applied_forces_ref.AppliedSim(ref, *blobs(env)) for _ in range(2))
    a_sim.reset_to(0, 17)
    b_sim.reset_to(0, 17)
    for _ in range(8):
        act = rng.uniform(-1, 1, m.nu)
        ctrl = np.zeros(m.nu)
        ctrl[spec.act_idx] = act * spec.act_delta + spec.act_mean
        qfrc = np.zeros(m.nv)
        qfrc[dof] = gear * gain * np.clip(ctrl, rng_[:, 0], rng_[:, 1])
        qa, va = a_sim.env_step(act)
        qb, vb = b_sim.env_step(np.zeros(m.nu), qfrc=qfrc)
        assert np.allclose(qa, qb, rtol=1e-9, atol=1e-9) and np.allclose(va, vb, rtol=1e-8, atol=1e-8), \
            (np.abs(qa - qb).max(), np.abs(va - vb).max())
    a_sim.close()
    b_sim.close()


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "HumanoidTorque.run"])
def test_zero_forces_leave_the_oracle_step_unchanged(ref, bundled_only, task):
    """zero buffers, and no buffers, step bit for bit like the oracle's own ref_step"""
    env = make_env(task)
    rng = np.random.RandomState(3)
    sims = [applied_forces_ref.AppliedSim(ref, *blobs(env)) for _ in range(3)]
    for s in sims:
        s.reset_to(0, 5)
    nb, nv, nu = sims[0].nb, sims[0].nv, env._model.nu
    for _ in range(5):
        act = rng.uniform(-1, 1, nu)
        qa, va = sims[0].env_step(act, xfrc=np.zeros((nb, 6)), qfrc=np.zeros(nv))
        qb, vb = sims[1].env_step(act)
        sims[2].oe.step(act)
        qc, vc = sims[2].get_state()
        assert np.array_equal(qa, qc) and np.array_equal(va, vc)
        assert np.array_equal(qb, qc) and np.array_equal(vb, vc)
    for s in sims:
        s.close()


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "HumanoidTorque.run", "Atlas.walk", "Talos.walk", "Atlas.walk+arms"])
def test_serial_core_matches_the_reference(emu, ref, bundled_only, task):
    """The serial build of the CUDA core (same source as the kernels) with random wrenches on random bodies and random joint
    forces against the fp64 reference, within the tolerance of test_core_emulation (2e-3 on the state)."""
    from loco_mujoco_b200 import modelpack
    applied_forces_ref.emu_bind_applied(emu)
    env = make_variant(task)
    m, spec = env._model, env.task_spec()
    ints, reals = modelpack.pack(m)
    p = applied_forces_ref._p
    sim = emu.emu_create(p(ints), len(ints), p(reals), len(reals))
    assert sim
    oe = applied_forces_ref.AppliedSim(ref, *blobs(env))
    rng = np.random.RandomState(4)
    q, v = np.zeros(m.nv), np.zeros(m.nv)
    oe.reset_to(0, 11)
    q[:], v[:] = oe.get_state()
    emu.emu_reset(sim, p(q), p(v))
    xf = np.zeros((m.nbody, 6), dtype=np.float32)
    qf = np.zeros(m.nv, dtype=np.float32)
    emu.emu_set_applied(sim, p(xf), p(qf))
    worst, acts = 0.0, []
    for k in range(6):
        xf[:] = 0
        for b in rng.choice(np.arange(1, m.nbody), size=2, replace=False):
            xf[b] = rng.randn(6) * [30, 30, 30, 3, 3, 3]
        qf[:] = rng.randn(m.nv) * 2.0
        a = rng.randn(m.nu) * 0.1
        acts.append(a)
        ctrl = np.zeros(m.nu)
        ctrl[spec.act_idx] = a * spec.act_delta + spec.act_mean
        emu.emu_step(sim, p(ctrl), spec.n_substeps)
        emu.emu_get_state(sim, p(q), p(v))
        qo, vo = oe.env_step(a, xfrc=xf.astype(np.float64), qfrc=qf.astype(np.float64))
        worst = max(worst, float(np.abs(q - qo).max()), float(np.abs(v - vo).max()))
    emu.emu_destroy(sim)
    # the forces must have changed the trajectory (else the comparison says nothing)
    plain = applied_forces_ref.AppliedSim(ref, *blobs(env))
    plain.reset_to(0, 11)
    for a in acts:
        qp, vp = plain.env_step(a)
    moved = float(np.abs(vp - vo).max())
    oe.close()
    plain.close()
    assert worst < 2e-3, "serial core drifted %.3e from the fp64 reference" % worst
    assert moved > 1e-2, moved


# ---------------------------------------------------------------------------------------------------------------------
# host logic
# ---------------------------------------------------------------------------------------------------------------------
def test_body_index(bundled_only):
    env = make_env("UnitreeA1.simple")
    names = env._model.body_names
    assert env.body_index("trunk") == names.index("trunk") > 0
    with pytest.raises(ValueError, match="unknown body"):
        env.body_index("no_such_body")


def test_body_index_names_the_parent_of_a_fused_body(tmp_path):
    from loco_mujoco_b200 import mjcf
    xml = tmp_path / "m.xml"
    xml.write_text("""<mujoco><worldbody>
      <body name="base" pos="0 0 1"><joint name="root_z" type="slide" axis="0 0 1"/>
        <geom type="sphere" size="0.1" mass="1"/>
        <body name="plate" pos="0 0 0.2"><geom type="box" size="0.1 0.1 0.01" mass="0.5"/>
          <body name="sensor" pos="0 0 0.05"><geom type="sphere" size="0.01" mass="0.01"/></body></body>
        <body name="arm" pos="0.2 0 0"><joint name="elbow" type="hinge" axis="0 1 0"/>
          <geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.03" mass="0.3"/></body>
      </body></worldbody></mujoco>""")
    m = mjcf.compile_model(mjcf.XmlHandle(str(xml)))
    assert m.body_names == ["world", "base", "arm"]
    assert m.body_index("arm") == 2
    for name in ("plate", "sensor"):        # (sensor's parent was fused too: the message names the surviving body)
        with pytest.raises(ValueError, match="fused into 'base'"):
            m.body_index(name)
    with pytest.raises(ValueError, match="unknown body"):
        m.body_index("leg")
    from loco_mujoco_b200 import modelpack
    assert modelpack.from_npz_dict(modelpack.to_npz_dict(m)).fused_bodies == m.fused_bodies


class _FakeTensor:
    def __init__(self, shape, dtype="float32", contiguous=True, device="cuda:0"):
        self.shape, self.dtype, self._c, self.device = shape, dtype, contiguous, device

    def is_contiguous(self):
        return self._c


def test_set_applied_forces_validates_its_arguments():
    """shape / dtype / layout checks happen before the engine is called (no device needed)"""
    import types
    from loco_mujoco_b200.engine import CudaEngine
    calls = []
    eng = object.__new__(CudaEngine)
    eng.torch = types.SimpleNamespace(float32="float32")
    eng.n_envs, eng.nbody, eng.nq, eng.device, eng.h = 4, 3, 5, "cuda:0", None
    eng.lib = types.SimpleNamespace(locosim_set_applied_forces=lambda h, x, q: calls.append((x, q)) or 0)
    import loco_mujoco_b200.engine as engine_mod
    orig = engine_mod._ptr
    engine_mod._ptr = lambda t: None if t is None else id(t)
    try:
        ok_x, ok_q = _FakeTensor((4, 3, 6)), _FakeTensor((4, 5))
        eng.set_applied_forces(ok_x, ok_q)
        eng.set_applied_forces(None, ok_q)
        eng.set_applied_forces()
        assert calls == [(id(ok_x), id(ok_q)), (None, id(ok_q)), (None, None)]
        for bad in (_FakeTensor((4, 3, 7)), _FakeTensor((3, 3, 6)), _FakeTensor((4, 3, 6), dtype="float64"),
                    _FakeTensor((4, 3, 6), contiguous=False), _FakeTensor((4, 3, 6), device="cuda:1")):
            with pytest.raises(ValueError):
                eng.set_applied_forces(bad, None)
        with pytest.raises(ValueError):
            eng.set_applied_forces(None, _FakeTensor((4, 6)))
        assert len(calls) == 3
    finally:
        engine_mod._ptr = orig


def test_4ages_all_refuses_applied_forces(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    env = LocoEnv.make("HumanoidTorque4Ages.walk.all.real", num_envs=8, debug=True)
    for get in (lambda: env.xfrc_applied, lambda: env.qfrc_applied, lambda: env.body_index("torso")):
        with pytest.raises(NotImplementedError):
            get()
