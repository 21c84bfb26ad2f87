"""Dynamics terms (include/locosim.h locosim_dynamics_terms: M, qfrc_bias, qfrc_passive, the centre of mass, mj_jacBody at
xpos, mj_jacSubtreeCom) without a GPU: the fp64 reference (tests/dynamics_terms_ref.py) on scenes with closed-form answers and
against physical identities for every bundled model, the serial build of the CUDA core against that reference for every
kernel configuration, and the host-side rules."""
import types

import numpy as np
import pytest

import dynamics_terms_ref as dtr
from full_body import make_variant
from position_mode import compile_xml, make_position

# one task per kernel configuration (locosim_host.h select_cfg)
CFG_TASKS = {"CfgEllEuler": "UnitreeA1.simple", "CfgPyrEuler": "Talos.walk", "CfgPyrRK4": "HumanoidTorque.run",
             "CfgPyrEuler29": "UnitreeH1.walk+arms", "CfgPyrRK4_31": "Atlas.walk+arms", "CfgPyrEuler31": "Talos.walk+arms"}
# every bundled model: the configurations' tasks, UnitreeA1 under position control, the models without arms, the four
# HumanoidTorque4Ages humanoids and the carry tasks (every carried weight's model)
IDENTITY_TASKS = list(CFG_TASKS.values()) + ["UnitreeA1.simple+position", "UnitreeG1.walk", "Atlas.walk", "UnitreeH1.walk",
                                             "HumanoidTorque4Ages.walk.1", "HumanoidTorque4Ages.walk.2",
                                             "HumanoidTorque4Ages.walk.3", "HumanoidTorque4Ages.walk.4", "Atlas.carry",
                                             "Talos.carry", "UnitreeH1.carry"]
G = 9.81


@pytest.fixture(scope="module")
def ref():
    return dtr.load()


def make_task(task, **kw):
    """make_variant for the task names above ("UnitreeA1.<task>+position": action_mode "position")"""
    if task.endswith("+position"):
        return make_position(task[:-len("+position")], **kw)
    return make_variant(task, **kw)


def _emu(emu, packed):
    dtr.emu_bind(emu)
    ints, reals = np.ascontiguousarray(packed[0], dtype=np.int32), np.ascontiguousarray(packed[1], dtype=np.float64)
    s = emu.emu_create(dtr._p(ints), len(ints), dtr._p(reals), len(reals))
    assert s
    return s


def _samples(env, n, seed, vel_scale=0.0):
    """n reset-table states (qpos, qvel) of env; qvel plus normal noise of vel_scale"""
    spec = env.task_spec()
    table = spec.table.reshape(-1, spec.table.shape[-1])
    nv = env._model.nv
    rng = np.random.RandomState(seed)
    out = []
    for i in rng.randint(len(table), size=n):
        q, v = table[i, :nv].astype(np.float64), table[i, nv:2 * nv].astype(np.float64)
        out.append((q, v + vel_scale * rng.normal(size=nv)))
    return out


def _quat2mat(q):
    w, x, y, z = q
    return np.array([[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]])


# ---------------------------------------------------------------------------------------------------------------------
# analytic scenes
# ---------------------------------------------------------------------------------------------------------------------
# a hinge pendulum about y with its CoM l below the axis, armature, stiffness, damping and a spring reference; a tip body
# (its own mass at its origin) L below the axis
M1, L1, IYY1, M2, L2, IYY2, ARM, K, B, QS = 2.0, 0.3, 0.05, 0.5, 0.8, 0.01, 0.07, 3.0, 0.4, 0.2
PENDULUM_XML = """
<mujoco model="pendulum">
  <compiler angle="radian"/>
  <option timestep="0.002" integrator="Euler"/>
  <worldbody>
    <body name="arm" pos="0 0 1">
      <joint name="h" type="hinge" axis="0 1 0" armature="%g" stiffness="%g" damping="%g" springref="%g"/>
      <inertial pos="0 0 -%g" mass="%g" diaginertia="0.02 %g 0.03"/>
      <body name="tip" pos="0 0 -%g">
        <inertial pos="0 0 0" mass="%g" diaginertia="0.004 %g 0.006"/>
      </body>
    </body>
  </worldbody>
</mujoco>
""" % (ARM, K, B, QS, L1, M1, IYY1, L2, M2, IYY2)

# a planar two-link arm about y without gravity: links of length l1 / l2 with their CoMs lc1 / lc2 along them
A_M1, A_M2, A_L1, A_LC1, A_LC2, A_I1, A_I2 = 1.5, 0.8, 0.6, 0.25, 0.3, 0.04, 0.02
ARM_XML = """
<mujoco model="two_link">
  <compiler angle="radian"/>
  <option timestep="0.002" integrator="Euler" gravity="0 0 0"/>
  <worldbody>
    <body name="l1" pos="0 0 2">
      <joint name="j1" type="hinge" axis="0 1 0"/>
      <inertial pos="0 0 -%g" mass="%g" diaginertia="0.01 %g 0.01"/>
      <body name="l2" pos="0 0 -%g">
        <joint name="j2" type="hinge" axis="0 1 0"/>
        <inertial pos="0 0 -%g" mass="%g" diaginertia="0.01 %g 0.01"/>
      </body>
    </body>
  </worldbody>
</mujoco>
""" % (A_LC1, A_M1, A_I1, A_L1, A_LC2, A_M2, A_I2)

SLIDE_XML = """
<mujoco model="slide">
  <option timestep="0.002" integrator="Euler"/>
  <worldbody>
    <body name="block" pos="0 0 0.5">
      <joint name="z" type="slide" axis="0 0 1" armature="0.1"/>
      <inertial pos="0 0 0.05" mass="3" diaginertia="0.01 0.01 0.01"/>
    </body>
  </worldbody>
</mujoco>
"""


def _both(emu, ref, xml, q, v):
    """(reference terms, serial-core terms) of a hand-built model at (q, v)"""
    m, packed = compile_xml(xml)
    r = dtr.DynRef(ref, m)
    s = _emu(emu, packed)
    want = r.terms(q, v)
    got = dtr.emu_terms(emu, s, m.nv, m.nbody, q, v)
    r.close()
    emu.emu_destroy(s)
    return want, got


@pytest.mark.parametrize("th,thd", [(0.0, 0.0), (0.7, -1.3), (-2.1, 2.5)])
def test_pendulum_in_closed_form(emu, ref, th, thd):
    want, got = _both(emu, ref, PENDULUM_XML, [th], [thd])
    M = IYY1 + M1 * L1 ** 2 + IYY2 + M2 * L2 ** 2 + ARM
    bias = (M1 * L1 + M2 * L2) * G * np.sin(th)
    passive = -K * (th - QS) - B * thd
    for k, x in (("M", M), ("bias", bias), ("passive", passive)):
        assert abs(want[k].ravel()[0] - x) < 1e-9 * (1 + abs(x)), (k, want[k], x)
        assert abs(float(got[k].ravel()[0]) - x) < 4e-6 * (1 + abs(x)), (k, got[k], x)
    com = (M1 * np.array([-L1 * np.sin(th), 0, 1 - L1 * np.cos(th)]) + M2 * np.array([-L2 * np.sin(th), 0, 1 - L2 * np.cos(th)]))
    com /= M1 + M2
    assert np.allclose(want["com"], list(com) + [M1 + M2], rtol=0, atol=1e-12)
    assert np.allclose(got["com"], list(com) + [M1 + M2], rtol=0, atol=1e-6)


def test_pendulum_tip_jacobian(emu, ref):
    th = 0.9
    want, got = _both(emu, ref, PENDULUM_XML, [th], [0.0])
    tip = np.array([0, 1, 0, -L2 * np.cos(th), 0, L2 * np.sin(th)])     # omega x (xpos - anchor) per unit rate, about y
    arm = np.array([0, 1, 0, 0, 0, 0])                                   # the arm's origin is on the axis
    for x in (want, got):
        assert np.allclose(x["jac"][2, :, 0], tip, atol=1e-6) and np.allclose(x["jac"][1, :, 0], arm, atol=1e-6)
        assert not np.any(x["jac"][0])
    assert np.array_equal(got["jac"][0], np.zeros((6, 1), np.float32))
    c = (M1 * L1 + M2 * L2) / (M1 + M2)
    for x in (want, got):
        assert np.allclose(x["jac_com"][:, 0], [-c * np.cos(th), 0, c * np.sin(th)], atol=1e-6)


@pytest.mark.parametrize("q2,qd1,qd2", [(0.0, 0.5, -0.3), (1.1, -2.0, 1.5), (-2.4, 0.7, 3.0)])
def test_two_link_arm_in_closed_form(emu, ref, q2, qd1, qd2):
    want, got = _both(emu, ref, ARM_XML, [0.4, q2], [qd1, qd2])
    c, s = np.cos(q2), np.sin(q2)
    M = np.array([[A_I1 + A_I2 + A_M1 * A_LC1 ** 2 + A_M2 * (A_L1 ** 2 + A_LC2 ** 2 + 2 * A_L1 * A_LC2 * c),
                   A_I2 + A_M2 * (A_LC2 ** 2 + A_L1 * A_LC2 * c)], [0, A_I2 + A_M2 * A_LC2 ** 2]])
    M[1, 0] = M[0, 1]
    h = A_M2 * A_L1 * A_LC2 * s
    cq = np.array([-h * (2 * qd1 * qd2 + qd2 ** 2), h * qd1 ** 2])       # C(q, qd) qd, no gravity
    assert np.allclose(want["M"], M, rtol=0, atol=1e-12) and np.allclose(want["bias"], cq, rtol=0, atol=1e-12)
    assert np.allclose(got["M"], M, rtol=0, atol=2e-6) and np.allclose(got["bias"], cq, rtol=0, atol=2e-5 * (1 + np.abs(cq).max()))
    assert not np.any(want["passive"]) and not np.any(got["passive"])


def test_slide_under_gravity(emu, ref):
    want, got = _both(emu, ref, SLIDE_XML, [0.25], [1.5])
    for x in (want, got):
        assert np.allclose(x["M"], [[3.1]], atol=1e-6) and np.allclose(x["bias"], [3 * G], rtol=1e-6)
        assert np.allclose(x["com"], [0, 0, 0.5 + 0.25 + 0.05, 3.0], atol=1e-6)
        assert np.allclose(x["jac"][1, :, 0], [0, 0, 0, 0, 0, 1], atol=1e-7)
        assert np.allclose(x["jac_com"][:, 0], [0, 0, 1], atol=1e-7)


# ---------------------------------------------------------------------------------------------------------------------
# identities on the reference, every bundled model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", IDENTITY_TASKS)
def test_identities_on_the_reference(ref, bundled_only, task):
    """M symmetric positive definite; bias(q, 0) = dV/dq, V = -sum m_b g . xipos_b (central differences); 1/2 v^T M v =
    the kinetic energy summed from the bodies' velocities (central differences of the frames along v); every carried
    weight's model of a carry task"""
    env = make_task(task)
    for mi, model in enumerate(env._models):
        r = dtr.DynRef(ref, model)
        g = np.array([0.0, 0.0, -G])
        iquat = np.asarray(model.body_iquat, dtype=np.float64).reshape(-1, 4)
        inertia = np.asarray(model.body_inertia, dtype=np.float64).reshape(-1, 3)
        for q, v in _samples(env, 3, 17 + mi, vel_scale=0.5):
            t = r.terms(q, np.zeros_like(v), jac=False)
            M = t["M"]
            assert np.array_equal(M, M.T) and np.linalg.eigvalsh(M).min() > 0, task
            h = 1e-6
            grad = np.zeros(r.nv)
            for d in range(r.nv):
                e = np.zeros(r.nv)
                e[d] = h
                V1 = -(r.mass * (r.frames(q + e)[2] @ g)).sum()
                V0 = -(r.mass * (r.frames(q - e)[2] @ g)).sum()
                grad[d] = (V1 - V0) / (2 * h)
            assert np.allclose(t["bias"], grad, rtol=1e-6, atol=1e-6 * max(1.0, np.abs(grad).max())), (task, t["bias"] - grad)
            # kinetic energy from body velocities
            eps = 1e-6
            _, xq1, xi1 = r.frames(q + eps * v)
            _, xq0, xi0 = r.frames(q - eps * v)
            _, xq, _ = r.frames(q)
            ke = 0.0
            for b in range(1, r.nb):
                vb = (xi1[b] - xi0[b]) / (2 * eps)
                dq = dtr.quat_mul(xq1[b], xq0[b] * np.array([1.0, -1.0, -1.0, -1.0]))
                w = dq[1:] * np.sign(dq[0]) / eps
                R = _quat2mat(dtr.quat_mul(xq[b], iquat[b]))
                ke += 0.5 * r.mass[b] * vb @ vb + 0.5 * w @ (R @ np.diag(inertia[b]) @ R.T) @ w
            tv = r.terms(q, v, jac=False)
            arm = np.asarray(model.dof_armature, dtype=np.float64)
            ke_m = 0.5 * v @ (tv["M"] - np.diag(arm)) @ v                   # (armature is rotor inertia, not a body's)
            assert abs(ke_m - ke) <= 1e-6 * max(1.0, ke), (task, ke_m, ke)
        r.close()


# ---------------------------------------------------------------------------------------------------------------------
# the serial fp32 core against the fp64 reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", list(CFG_TASKS))
def test_serial_core_matches_the_reference(emu, ref, bundled_only, cfg):
    """emu_dynamics_terms (the kernels' source, serial) at 20 reset-table states with perturbed velocities, every term
    within dynamics_terms_ref's fp32 error model, at the fp32-rounded state the core sees"""
    from loco_mujoco_b200 import modelpack
    env = make_task(CFG_TASKS[cfg])
    m = env._model
    s = _emu(emu, modelpack.pack(m))
    r = dtr.DynRef(ref, m)
    worst = {}
    for q, v in _samples(env, 20, 23, vel_scale=1.0):
        q32, v32 = q.astype(np.float32), v.astype(np.float32)
        got = dtr.emu_terms(emu, s, m.nv, m.nbody, q32, v32)
        want = r.terms(q32.astype(np.float64), v32.astype(np.float64))
        for k, x in dtr.check(got, want).items():
            worst[k] = max(worst.get(k, 0.0), x)
    r.close()
    emu.emu_destroy(s)
    print("%s: largest error / bound per term: %s" % (cfg, ", ".join("%s %.3g" % kv for kv in sorted(worst.items()))))


def test_non_finite_state_gives_zero_rows(emu):
    m, packed = compile_xml(ARM_XML)
    s = _emu(emu, packed)
    for q, v in (([np.nan, 0.1], [0, 0]), ([0.2, 0.1], [0, np.inf])):
        got = dtr.emu_terms(emu, s, m.nv, m.nbody, np.array(q), np.array(v))
        for k in dtr.TERMS:
            assert np.array_equal(got[k], np.zeros_like(got[k])), k
    got = dtr.emu_terms(emu, s, m.nv, m.nbody, np.array([0.2, 0.1]), np.array([0.3, 0.0]))
    assert all(np.isfinite(got[k]).all() for k in dtr.TERMS) and got["M"][0, 0] > 0
    emu.emu_destroy(s)


def test_outputs_left_null_are_not_written(emu):
    m, packed = compile_xml(PENDULUM_XML)
    s = _emu(emu, packed)
    emu.emu_reset(s, dtr._p(np.array([0.3])), dtr._p(np.array([0.1])))
    com = np.full(4, np.nan, np.float32)
    emu.emu_dynamics_terms(s, None, None, None, com.ctypes.data_as(dtr.ctypes.c_void_p), None, None)
    assert np.isfinite(com).all() and abs(com[3] - (M1 + M2)) < 1e-6
    emu.emu_destroy(s)


# ---------------------------------------------------------------------------------------------------------------------
# host logic
# ---------------------------------------------------------------------------------------------------------------------
class _FakeTensor:
    def __init__(self, shape, dtype="float32", contiguous=True, device="cuda:0", ptr=0):
        self.shape, self.dtype, self._c, self.device, self._ptr = shape, dtype, contiguous, device, ptr

    def is_contiguous(self):
        return self._c

    def data_ptr(self):
        return self._ptr


def test_dynamics_terms_validates_its_arguments(monkeypatch):
    """dtype / shape / layout / device / overlap checks happen before the engine is called (no device needed); nothing
    is launched when no output is given"""
    from loco_mujoco_b200 import engine as engine_mod
    calls = []
    eng = object.__new__(engine_mod.CudaEngine)
    eng.torch = types.SimpleNamespace(float32="float32", Tensor=_FakeTensor)
    eng.n_envs, eng.nq, eng.nbody, eng.device, eng.h, eng.launches = 4, 18, 14, "cuda:0", None, 0
    eng.lib = types.SimpleNamespace(locosim_dynamics_terms=lambda h, *a: calls.append(a) or 0)
    eng._stream = lambda: None
    monkeypatch.setattr(engine_mod, "_ptr", lambda t: None if t is None else id(t))
    shapes = dict(M=(4, 18, 18), bias=(4, 18), passive=(4, 18), com=(4, 4), jac=(4, 14, 6, 18), jac_com=(4, 3, 18))
    base, good = 1 << 30, {}
    for k, sh in shapes.items():
        good[k] = _FakeTensor(sh, ptr=base)
        base += 4 * int(np.prod(sh))
    assert eng.dynamics_terms() == {} and calls == []
    assert eng.dynamics_terms(**good) == good and len(calls) == 1 and eng.launches == 1
    assert eng.dynamics_terms(com=good["com"]) == {"com": good["com"]} and calls[-1][:3] == (None, None, None)
    for k, sh in shapes.items():
        bad = [_FakeTensor(sh[:-1] + (sh[-1] + 1,)), _FakeTensor((5,) + sh[1:]), _FakeTensor(sh, "float64"),
               _FakeTensor(sh, contiguous=False), _FakeTensor(sh, device="cuda:1"), np.zeros(sh, np.float32)]
        for x in bad:
            with pytest.raises(ValueError):
                eng.dynamics_terms(**dict(good, **{k: x}))
    # overlapping outputs are refused: the last float of one tensor shared with the first of the next
    for k1, k2 in (("M", "bias"), ("bias", "jac"), ("jac", "jac_com"), ("com", "M")):
        a = _FakeTensor(shapes[k1], ptr=1 << 20)
        b = _FakeTensor(shapes[k2], ptr=(1 << 20) + 4 * int(np.prod(shapes[k1])) - 4)
        with pytest.raises(ValueError, match="overlap"):
            eng.dynamics_terms(**{k1: a, k2: b})
    assert len(calls) == 2


def test_4ages_all_refuses_dynamics_terms(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    env = LocoEnv.make("HumanoidTorque4Ages.walk.all.real", num_envs=8, debug=True)
    with pytest.raises(NotImplementedError):
        env.dynamics_terms()
    with pytest.raises(NotImplementedError):
        env.dynamics_terms(body_jacobian=True, out={})
