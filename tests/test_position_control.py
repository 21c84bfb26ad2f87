"""UnitreeA1 under PD position control (action_mode "position" / "position_difference") without a GPU: the MJCF <position>
actuator, the host rules of the action modes, and the physics of position actuators on the fp64 oracle, read through the
dof outputs' reference (tests/dof_outputs_ref.py)."""

import numpy as np
import pytest
from scipy.optimize import brentq

import dof_outputs_ref as dor
from helpers import blobs
from position_mode import CTRLRANGE, FORCE, KP, Sim, compile_xml, make_position


@pytest.fixture(scope="module")
def ref():
    return dor.load()


def _check_a1_actuators(m):
    assert m.nu == 12
    assert np.array_equal(m.actuator_gain, np.full(12, KP))
    assert np.array_equal(m.actuator_bias, np.tile([0.0, -KP, 0.0], (12, 1)))
    assert np.array_equal(m.actuator_gear, np.ones(12))
    assert m.actuator_ctrllimited.all() and m.actuator_forcelimited.all()
    assert np.array_equal(m.actuator_forcerange, np.tile([-FORCE, FORCE], (12, 1)))
    for i, name in enumerate(m.actuator_names):
        assert np.array_equal(m.actuator_ctrlrange[i], CTRLRANGE[name.split("_")[1]]), name
        assert m.jnt_names[m.actuator_dof[i]] == name + "_joint"


def test_position_fixture_has_the_position_actuators(bundled_only):
    env = make_position()
    _check_a1_actuators(env._model)


def test_position_xml_compiles_like_mujoco(monkeypatch):
    """the reference's unitree_a1_position.xml through the parser: kp / forcerange inherited from class a1, ctrlrange from
    abduction / hip / knee; the compiled model is the shipped fixture, bit for bit"""
    from loco_mujoco_b200 import modelpack
    from loco_mujoco_b200.environments.base import reference_data_root
    monkeypatch.delenv("LOCO_MUJOCO_B200_FORCE_BUNDLED", raising=False)
    if reference_data_root() is None:
        pytest.skip("no loco_mujoco checkout (LOCO_MUJOCO_PATH)")
    live = make_position()
    _check_a1_actuators(live._model)
    monkeypatch.setenv("LOCO_MUJOCO_B200_FORCE_BUNDLED", "1")
    fixture = make_position()
    for a, b in zip(modelpack.pack(live._model), modelpack.pack(fixture._model)):
        assert np.array_equal(a, b)


HINGE_XML = """
<mujoco model="pendulum">
  <compiler angle="radian"/>
  <option timestep="0.002" integrator="Euler"/>
  <worldbody>
    <body name="arm" pos="0 0 1">
      <joint name="j" type="hinge" axis="0 1 0" damping="3"{range}/>
      <geom name="bob" type="sphere" size="0.02" pos="0 0 -{l}" mass="{m}" contype="0" conaffinity="0"/>
    </body>
  </worldbody>
  <actuator>
    <position name="p" joint="j" kp="{kp}" ctrllimited="true" ctrlrange="{ctrl}" forcelimited="true" forcerange="{force}"{extra}/>
  </actuator>
</mujoco>
"""


def _hinge(kp=10.0, m=1.0, l=0.5, ctrl="-3 3", force="-100 100", rng="", extra=""):
    return HINGE_XML.format(kp=kp, m=m, l=l, ctrl=ctrl, force=force, range=rng, extra=extra)


def test_position_actuator_compiles_gain_and_bias():
    m, _ = compile_xml(_hinge(kp=7.5))
    assert m.actuator_gain[0] == 7.5 and np.array_equal(m.actuator_bias[0], [0, -7.5, 0])
    assert m.actuator_ctrllimited[0] == 1 and m.actuator_forcelimited[0] == 1
    m, _ = compile_xml(_hinge().replace(' kp="10.0"', ""))        # MuJoCo's default kp
    assert m.actuator_gain[0] == 1.0 and np.array_equal(m.actuator_bias[0], [0, -1, 0])


def test_position_actuator_rules():
    # the engine evaluates the bias at qpos / qvel of the dof: a gear would need the actuator length gear * qpos
    with pytest.raises(NotImplementedError, match="gear"):
        compile_xml(_hinge(extra=' gear="2"'))
    # the only joints the parser builds are hinges and slides: a ball joint is refused before any actuator is read
    with pytest.raises(NotImplementedError, match="joint type ball"):
        compile_xml(_hinge().replace('type="hinge" axis="0 1 0"', 'type="ball"'))
    for tag in ("velocity", "intvelocity", "cylinder", "muscle"):
        with pytest.raises(NotImplementedError, match="actuator <%s>" % tag):
            compile_xml(_hinge().replace("<position", "<" + tag).replace(' kp="10.0"', ""))


def test_action_mode_validation(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    from loco_mujoco_b200.environments.unitree_a1 import UnitreeA1
    for bad in ("velocity", "Position", None):
        with pytest.raises(ValueError, match="action_mode"):
            LocoEnv.make("UnitreeA1.simple.real", debug=True, action_mode=bad)
    with pytest.raises(ValueError, match="action_mode"):
        UnitreeA1(action_mode="pd")


def test_missing_position_asset_is_an_error(bundled_only, monkeypatch):
    """without a checkout and without the fixture directory the position model is missing: never the torque model instead"""
    monkeypatch.delenv("LOCO_MUJOCO_B200_ASSET_PATH")
    with pytest.raises(FileNotFoundError, match=r"UnitreeA1\.simple\+position"):
        make_position()
    with pytest.raises(FileNotFoundError, match=r"UnitreeA1\.hard\+position"):
        make_position("UnitreeA1.hard", mode="position_difference")


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "UnitreeA1.hard"])
def test_both_position_modes_build_the_same_engine_inputs(bundled_only, task):
    a, b = make_position(task, "position"), make_position(task, "position_difference")
    for x, y in zip(blobs(a), blobs(b)):
        for u, v in zip(x, y):
            assert np.array_equal(u, v)
    torque = make_position(task, "torque")
    assert not np.array_equal(blobs(a)[0][1], blobs(torque)[0][1])


def test_action_normalisation_spans_each_ctrlrange(bundled_only):
    env = make_position()
    spec, m = env.task_spec(), env._model
    lo, hi = spec.act_mean - spec.act_delta, spec.act_mean + spec.act_delta
    for k, i in enumerate(spec.act_idx):
        assert np.allclose([lo[k], hi[k]], m.actuator_ctrlrange[i], rtol=0, atol=1e-12), m.actuator_names[i]


def test_position_mode_selects_the_torque_models_configuration(emu, bundled_only):
    from loco_mujoco_b200 import modelpack
    cfgs = []
    for mode in ("torque", "position"):
        ints, reals = [np.ascontiguousarray(x) for x in modelpack.pack(make_position(mode=mode)._model)]
        ints, reals = ints.astype(np.int32), reals.astype(np.float64)
        cfgs.append(emu.emu_select_cfg(dor._p(ints), len(ints), dor._p(reals), len(reals)))
    assert cfgs[0] == cfgs[1] >= 0


# ---------------------------------------------------------------------------------------------------------------------
# physics of position actuators on the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------------
def test_hinge_settles_where_the_actuator_balances_gravity(ref):
    """a pendulum (point mass m at distance l) under <position kp>: at rest kp (target - q) = m g l sin q, and qfrc_actuator
    is the analytic clamp at the evaluation state"""
    kp, mass, l, g, target = 10.0, 1.0, 0.5, 9.81, 0.8
    _, packed = compile_xml(_hinge(kp=kp, m=mass, l=l))
    sim = Sim(ref, packed)
    sim.reset([0.0], [0.0])
    for _ in range(40):
        dor.step(ref, sim.sim, [target], 100)
    q, v = sim.state()
    want = brentq(lambda x: kp * (target - x) - mass * g * l * np.sin(x), 0.0, target)
    assert abs(v[0]) < 1e-9 and abs(q[0] - want) < 1e-7, (q, v, want)
    ref.lib.ref_forward(sim.sim, dor._p(np.array([target])))
    d = dor.now(ref, sim.sim)
    assert abs(d[0, 0] - kp * (target - q[0])) < 1e-12
    assert abs(d[0, 0] - mass * g * l * np.sin(q[0])) < 1e-6
    assert d[0, 1] == 0.0 and abs(d[0, 2]) < 1e-6               # no constraints, at rest
    # at other states and controls: clip(kp (clip(ctrl) - q), forcerange)
    rng = np.random.RandomState(0)
    for _ in range(20):
        q0, v0, c = rng.uniform(-2, 2), rng.uniform(-3, 3), rng.uniform(-5, 5)
        sim.reset([q0], [v0])
        ref.lib.ref_forward(sim.sim, dor._p(np.array([c])))
        want = np.clip(kp * (np.clip(c, -3, 3) - q0), -100, 100)
        assert abs(dor.now(ref, sim.sim)[0, 0] - want) < 1e-12
    sim.close()


def test_far_target_saturates_at_the_forcerange(ref):
    _, packed = compile_xml(_hinge(kp=10.0, force="-2 1.5"))
    sim = Sim(ref, packed)
    for q0, c, want in ((0.0, 3.0, 1.5), (0.0, -3.0, -2.0), (0.0, 50.0, 1.5), (2.5, -50.0, -2.0)):
        sim.reset([q0], [0.0])
        ref.lib.ref_forward(sim.sim, dor._p(np.array([c])))
        assert dor.now(ref, sim.sim)[0, 0] == want
    sim.close()


def test_a1_position_actuator_forces_at_rest_from_a_mocap_sample(ref, bundled_only):
    """A1 in position mode reset from the mocap table: every leg dof's qfrc_actuator is the analytic clamp at the state of
    the evaluation, for targets inside and outside the clamp"""
    env = make_position()
    m, spec = env._model, env.task_spec()
    oe = ref.env(*blobs(env))
    rng = np.random.RandomState(4)
    n_sat = 0
    for k in range(6):
        oe.reset_to(0, 37 * k)
        q, v = oe.get_state()
        a = rng.uniform(-1, 1, m.nu) * (1.0 if k % 2 else 1.5)      # (1.5: past the ctrlrange, clamped)
        ctrl = np.zeros(m.nu)
        ctrl[spec.act_idx] = a * spec.act_delta + spec.act_mean
        ref.lib.ref_forward(oe.sim, dor._p(ctrl))
        d = dor.now(ref, oe.sim)
        want = np.zeros(m.nv)
        for i in range(m.nu):
            dof = m.actuator_dof[i]
            c = np.clip(ctrl[i], *m.actuator_ctrlrange[i])
            want[dof] = np.clip(KP * (c - q[dof]), -FORCE, FORCE)
        n_sat += int((np.abs(want) == FORCE).sum())
        assert np.abs(d[:, 0] - want).max() < 1e-12, (k, d[:, 0], want)
        assert np.array_equal(d[:6, 0], np.zeros(6))                 # the unactuated root
    assert n_sat > 0
    oe.close()


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "UnitreeA1.simple+position", "HumanoidTorque.run"])
def test_joint_space_balance(ref, bundled_only, task):
    """M qacc = qfrc_smooth + qfrc_constraint at one evaluation (qfrc_smooth = passive - bias + actuator + applied): what pins
    the meaning of the three components"""
    from full_body import make_variant
    env = make_position(task.split("+")[0]) if task.endswith("+position") else make_variant(task)
    m, spec = env._model, env.task_spec()
    oe = ref.env(*blobs(env))
    rng = np.random.RandomState(2)
    table = spec.table.reshape(-1, spec.table.shape[-1])
    n_con = 0
    for i in rng.randint(len(table), size=6):
        q, v = table[i, :m.nv], table[i, m.nv:2 * m.nv]
        ctrl = np.zeros(m.nu)
        ctrl[spec.act_idx] = rng.uniform(-1, 1, m.nu) * spec.act_delta + spec.act_mean
        f = oe.forward(q, v, ctrl, m.nbody)
        d = dor.now(ref, oe.sim)
        passive, act = dor.forces(ref, oe.sim)
        assert np.array_equal(d[:, 0], act) and np.array_equal(d[:, 2], f["qacc"])
        assert np.allclose(f["qfrc_smooth"], passive - f["bias"] + act, rtol=0, atol=1e-12 * (1 + np.abs(f["bias"]).max()))
        lhs, rhs = f["M"] @ d[:, 2], f["qfrc_smooth"] + d[:, 1]
        assert np.abs(lhs - rhs).max() < 1e-9 * (1 + np.abs(rhs).max()), np.abs(lhs - rhs).max()
        n_con += int(np.abs(d[:, 1]).max() > 1e-3)
    assert n_con >= 3, "too few states with constraint forces"
    oe.close()


def test_joint_limit_shows_in_qfrc_constraint(ref):
    """a position target past a joint limit drives the joint into it: at rest the limit's force holds the actuator and
    gravity, and appears on the dof in qfrc_constraint (no other constraint exists)"""
    _, packed = compile_xml(_hinge(kp=10.0, rng=' limited="true" range="-0.4 0.4"'))
    sim = Sim(ref, packed)
    sim.reset([0.0], [0.0])
    for _ in range(20):
        d = dor.step(ref, sim.sim, [1.5], 100)
    q, v = sim.state()
    assert abs(v[0]) < 1e-6 and 0.39 < q[0] < 0.41, (q, v)           # at the limit (soft: slightly past it)
    ref.lib.ref_forward(sim.sim, dor._p(np.array([1.5])))
    d = dor.now(ref, sim.sim)
    gravity = -1.0 * 9.81 * 0.5 * np.sin(q[0])
    assert d[0, 0] == pytest.approx(10.0 * (1.5 - q[0]), abs=1e-12)
    assert d[0, 1] < -1.0 and abs(d[0, 0] + d[0, 1] + gravity) < 1e-4, d
    sim.close()
