"""Inverse dynamics (MuJoCo 2.3.7's continuous-time mj_inverse, include/locosim.h locosim_inverse) without a GPU: the fp64
reference (tests/inverse_ref.py) on hand-built scenes and against the forward solver it inverts, the serial build of the CUDA
core against that reference for every kernel configuration, and the host-side rules."""
import types

import numpy as np
import pytest

import inverse_ref as ivr
from full_body import make_variant
from helpers import blobs
from position_mode import Sim, compile_xml, make_position

# one task per kernel configuration (locosim_host.h select_cfg)
CFG_TASKS = {"CfgEllEuler": "UnitreeA1.simple", "CfgPyrEuler": "Talos.walk", "CfgPyrRK4": "HumanoidTorque.run",
             "CfgPyrEuler29": "UnitreeH1.walk+arms", "CfgPyrRK4_31": "Atlas.walk+arms", "CfgPyrEuler31": "Talos.walk+arms"}


@pytest.fixture(scope="module")
def ref():
    return ivr.load()


def make_task(task, **kw):
    """make_variant for the task names above ("UnitreeA1.<task>+position": action_mode "position")"""
    if task.endswith("+position"):
        return make_position(task[:-len("+position")], **kw)
    return make_variant(task, **kw)


class _Bare:
    """the fp64 reference on a bare oracle sim of a hand-built model"""

    def __init__(self, ref, packed):
        self.s = Sim(ref, packed)
        self.lib, self.nv = ref.lib, self.s.nv

    def inverse(self, q, v, qacc):
        p = ivr._p
        self.s.reset(q, v)
        self.lib.refinv_forward(self.s.sim, None, None, None, None, None)
        out, cons, scale = np.zeros(self.nv), np.zeros(self.nv), np.zeros(self.nv)
        self.lib.refinv_inverse(self.s.sim, p(np.ascontiguousarray(qacc, dtype=np.float64)), p(out), p(cons), p(scale))
        return out, cons, scale

    def close(self):
        self.s.close()


def _emu(emu, packed):
    ivr.emu_bind(emu)
    ints, reals = [np.ascontiguousarray(x) for x in packed]
    ints, reals = ints.astype(np.int32), reals.astype(np.float64)
    s = emu.emu_create(ivr._p(ints), len(ints), ivr._p(reals), len(reals))
    assert s
    return s


def _emu_inverse(emu, s, q, v, qacc):
    p = ivr._p
    emu.emu_reset(s, p(np.ascontiguousarray(q, dtype=np.float64)), p(np.ascontiguousarray(v, dtype=np.float64)))
    out = np.full(len(q), np.nan, dtype=np.float32)
    emu.emu_inverse(s, p(np.ascontiguousarray(qacc, dtype=np.float64)), p(out))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# analytic scenes
# ---------------------------------------------------------------------------------------------------------------------
# a frictionless ball on three slides; with default solref / solimp
BALL_XML = """
<mujoco model="ball">
  <option timestep="0.002" integrator="Euler" cone="pyramidal"/>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 1" condim="1"/>
    <body name="ball" pos="0 0 0">
      <joint name="x" type="slide" axis="1 0 0"/><joint name="y" type="slide" axis="0 1 0"/>
      <joint name="z" type="slide" axis="0 0 1"/>
      <geom name="g" type="sphere" size="0.1" mass="3" condim="1"/>
    </body>
  </worldbody>
</mujoco>
"""
# a sprung, damped hinge with armature, without gravity: I qacc + k (q - q0) + b qd
HINGE_XML = """
<mujoco model="hinge">
  <compiler angle="radian"/>
  <option timestep="0.002" integrator="Euler" gravity="0 0 0"/>
  <worldbody>
    <body name="arm" pos="0 0 1">
      <joint name="h" type="hinge" axis="0 0 1" stiffness="7" damping="0.6" springref="0.25" armature="0.05"/>
      <inertial pos="0 0 0" mass="2" diaginertia="0.1 0.2 0.3"/>
      <geom name="g" type="sphere" size="0.05" contype="0" conaffinity="0"/>
    </body>
  </worldbody>
</mujoco>
"""


def test_a_body_held_still_above_the_floor_needs_its_weight(emu, ref):
    m, packed = compile_xml(BALL_XML)
    r, s = _Bare(ref, packed), _emu(emu, packed)
    q, v, a = np.array([0.3, -0.2, 1.0]), np.zeros(3), np.zeros(3)
    want = np.array([0.0, 0.0, 3 * 9.81])
    got, cons, _ = r.inverse(q, v, a)
    assert np.allclose(got, want, rtol=0, atol=1e-12) and not cons.any()
    assert np.allclose(_emu_inverse(emu, s, q, v, a), want, rtol=2e-7, atol=0)
    r.close()
    emu.emu_destroy(s)


def test_a_body_resting_in_the_floor_needs_its_weight_less_the_soft_contact_force(emu, ref):
    m, packed = compile_xml(BALL_XML)
    r, s = _Bare(ref, packed), _emu(emu, packed)
    depth = 0.004                        # deeper than solimp's width (0.001): impedance = dmax
    q, v, a = np.array([0.0, 0.0, 0.1 - depth]), np.zeros(3), np.zeros(3)
    # soft contact at qvel = qacc = 0 (mj_makeImpedance, mj_referenceConstraint): aref = -K imp (dist - margin),
    # jar = -aref, force = -jar / R, R = (1 - imp) diag / imp, diag = the ball's translational invweight0
    dmax, tc, dr = 0.95, 0.02, 1.0
    K = 1.0 / (dmax * dmax * tc * tc * dr * dr)
    imp, diag = dmax, float(m.geom_invweight0[1, 0])
    R = (1 - imp) * diag / imp
    f = K * imp * depth / R
    want = np.array([0.0, 0.0, 3 * 9.81 - f])
    got, cons, _ = r.inverse(q, v, a)
    assert np.allclose(cons, [0, 0, f], rtol=1e-12, atol=0)
    assert np.allclose(got, want, rtol=1e-12, atol=1e-9), (got, want)
    assert np.allclose(_emu_inverse(emu, s, q, v, a), want, rtol=0, atol=1e-5 * f)
    r.close()
    emu.emu_destroy(s)


def test_a_sprung_damped_hinge(emu, ref):
    m, packed = compile_xml(HINGE_XML)
    r, s = _Bare(ref, packed), _emu(emu, packed)
    for q0, v0, a0 in ((0.0, 0.0, 0.0), (0.7, -1.3, 2.5), (-1.1, 0.4, -3.0)):
        want = (0.3 + 0.05) * a0 + 7 * (q0 - 0.25) + 0.6 * v0
        got, _, _ = r.inverse([q0], [v0], [a0])
        assert abs(got[0] - want) < 1e-12 * max(1.0, abs(want))
        assert abs(_emu_inverse(emu, s, [q0], [v0], [a0])[0] - want) < 1e-6 * max(1.0, abs(want))
    r.close()
    emu.emu_destroy(s)


# ---------------------------------------------------------------------------------------------------------------------
# the fp64 reference against the forward solver it inverts
# ---------------------------------------------------------------------------------------------------------------------
def _samples(env, n, seed):
    """n reset-table states (qpos, qvel) of env"""
    spec = env.task_spec()
    table = spec.table.reshape(-1, spec.table.shape[-1])
    nv = env._model.nv
    rng = np.random.RandomState(seed)
    return [(table[i, :nv].astype(np.float64), table[i, nv:2 * nv].astype(np.float64)) for i in rng.randint(len(table), size=n)]


def _ctrl(env, rng):
    spec = env.task_spec()
    c = np.zeros(env._model.nu)
    c[spec.act_idx] = rng.uniform(-1, 1, env._model.nu) * spec.act_delta + spec.act_mean
    return c


# every bundled model: the kernel configurations' tasks, UnitreeA1 under position control, the models without arms, the four
# HumanoidTorque4Ages humanoids and the carry tasks (their first carried weight)
IDENTITY_TASKS = list(CFG_TASKS.values()) + ["UnitreeA1.simple+position", "UnitreeG1.walk", "Atlas.walk", "UnitreeH1.walk",
                                             "HumanoidTorque4Ages.walk.1", "HumanoidTorque4Ages.walk.2",
                                             "HumanoidTorque4Ages.walk.3", "HumanoidTorque4Ages.walk.4", "Atlas.carry",
                                             "Talos.carry", "UnitreeH1.carry"]


@pytest.mark.parametrize("task", IDENTITY_TASKS)
def test_forward_and_inverse_agree_on_the_reference(ref, bundled_only, task):
    """mjENBL_FWDINV: at the forward solution qfrc_inverse - qfrc_actuator - qfrc_applied is the solver's gradient, below its
    tolerance where it converged; at any qacc it equals the central-difference gradient of the solver's cost"""
    env = make_task(task)
    mb, tb = blobs(env)
    sim = ivr.InverseSim(ref, mb, tb, env._model_user_features[0], env._model.geom_type)
    nv, nu = sim.nv, sim.nu
    scale = 1.0 / (sim.meaninertia() * max(nv, 1))
    rng = np.random.RandomState(3)
    converged = 0
    for q, v in _samples(env, 5, 7):
        ctrl, qfrc = _ctrl(env, rng), rng.normal(0, 5, nv)
        qacc, act, it = sim.forward(q, v, ctrl, qfrc=qfrc)
        res = sim.inverse(qacc)["qfrc"] - act - qfrc
        if it < env._model.opt_iterations:
            converged += 1
            assert scale * np.linalg.norm(res) < 1e-6, (task, it, scale * np.linalg.norm(res))
        # arbitrary qacc: the residual is the gradient of Gauss + constraint cost (signs, cone zones)
        qa = qacc + rng.normal(0, 1, nv) * (1 + np.abs(qacc))
        res = sim.inverse(qa)["qfrc"] - act - qfrc
        h = 1e-6 * (1 + np.abs(qa))
        grad = np.zeros(nv)
        for d in range(nv):
            e = np.zeros(nv)
            e[d] = h[d]
            grad[d] = (sim.cost(qa + e) - sim.cost(qa - e)) / (2 * h[d])
        assert np.allclose(res, grad, rtol=1e-5, atol=1e-5 * max(1.0, np.abs(grad).max())), (task, res - grad)
    sim.close()
    assert converged >= 3


# ---------------------------------------------------------------------------------------------------------------------
# the serial fp32 core against the fp64 reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", list(CFG_TASKS))
def test_serial_core_matches_the_reference(emu, ref, bundled_only, cfg):
    """emu_inverse (the kernels' source, serial) at reset-table states, at the reference's forward qacc of random controls
    and at perturbations of it, within c 2^-23 S_d per dof; samples that fail the bound must be explained by the reference
    (a contact set that changes at fp32 resolution, or an error within 10x the reference's own jump there) and are
    counted: at most 5 % of the samples, at least one"""
    from loco_mujoco_b200 import modelpack
    env = make_task(CFG_TASKS[cfg])
    mb, tb = blobs(env)
    m = env._model
    s = _emu(emu, modelpack.pack(m))
    assert emu.emu_select_cfg is not None
    sim = ivr.InverseSim(ref, mb, tb, env._model_user_features[0], m.geom_type)
    rng = np.random.RandomState(5)
    n, ambiguous, constrained = 0, 0, 0
    for q, v in _samples(env, 10, 11):
        qacc, act, _ = sim.forward(q, v, _ctrl(env, rng))
        for qa in (qacc, qacc + rng.normal(0, 0.5, m.nv) * (1 + np.abs(qacc))):
            got = _emu_inverse(emu, s, q.astype(np.float32), v.astype(np.float32), qa.astype(np.float32))
            # the reference at the fp32-rounded inputs the core sees
            want = sim.at(q.astype(np.float32), v.astype(np.float32), qa.astype(np.float32))
            n += 1
            constrained += int(np.abs(want["constraint"]).max() > 1.0)
            ok, ratio = ivr.within(got, want["qfrc"], want["scale"])
            if not ok:
                q32, v32, a32 = (x.astype(np.float32).astype(np.float64) for x in (q, v, qa))
                assert sim.explained(q32, v32, a32, got, want["qfrc"]), (cfg, ratio, got - want["qfrc"])
                ambiguous += 1
    sim.close()
    emu.emu_destroy(s)
    print("%s: %d of %d samples outside the bound, each explained by the reference" % (cfg, ambiguous, n))
    assert ambiguous <= ivr.allowed(n), (cfg, ambiguous, n)
    assert constrained >= 1, cfg


@pytest.mark.parametrize("cfg", ["CfgEllEuler", "CfgPyrRK4", "CfgPyrEuler31"])
def test_serial_core_inverts_its_own_forward_solution(emu, bundled_only, cfg):
    """emu_forward, then emu_inverse at its qacc: the actuator force, up to the fp32 solver's tolerance"""
    from loco_mujoco_b200 import modelpack
    env = make_task(CFG_TASKS[cfg])
    m = env._model
    s = _emu(emu, modelpack.pack(m))
    p = ivr._p
    rng = np.random.RandomState(2)
    gear = np.zeros(m.nv)
    for q, v in _samples(env, 4, 13):
        ctrl = _ctrl(env, rng)
        emu.emu_reset(s, p(q), p(v))
        emu.emu_set_ws(s, p(np.zeros(m.nv)))
        emu.emu_forward(s, p(ctrl))
        qacc = np.zeros(m.nv)
        emu.emu_get_qacc(s, p(qacc))
        out = np.zeros(m.nv, dtype=np.float32)
        emu.emu_inverse(s, p(qacc), p(out))
        # the actuator force of the evaluation (every actuator here has a constant gain and no bias but UnitreeA1's
        # position variant, which is not among these)
        act = np.zeros(m.nv)
        for i in range(m.nu):
            c = ctrl[i]
            if m.actuator_ctrllimited[i]:
                c = np.clip(c, *m.actuator_ctrlrange[i])
            f = m.actuator_gain[i] * c
            if m.actuator_forcelimited[i]:
                f = np.clip(f, *m.actuator_forcerange[i])
            act[m.actuator_dof[i]] += m.actuator_gear[i] * f
        scale = 1.0 / (float(m.stat_meaninertia) * m.nv)
        assert scale * np.linalg.norm(out - act) < 1e-3, (cfg, scale * np.linalg.norm(out - act))
    emu.emu_destroy(s)


def test_non_finite_input_gives_a_zero_row(emu, ref):
    m, packed = compile_xml(BALL_XML)
    s = _emu(emu, packed)
    q, v, a = np.array([0.0, 0.0, 0.05]), np.zeros(3), np.zeros(3)
    for qq, vv, aa in ((q, v, [0, np.nan, 0]), ([np.inf, 0, 0.05], v, a), (q, [0, 0, np.nan], a)):
        assert np.array_equal(_emu_inverse(emu, s, np.array(qq, float), np.array(vv, float), np.array(aa, float)), np.zeros(3))
    assert _emu_inverse(emu, s, q, v, a)[2] != 0.0
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


def test_inverse_validates_its_arguments(monkeypatch):
    """dtype / shape / layout / device / overlap checks happen before the engine is called (no device needed)"""
    from loco_mujoco_b200 import engine as engine_mod
    calls = []
    eng = object.__new__(engine_mod.CudaEngine)
    eng.torch = types.SimpleNamespace(float32="float32", Tensor=_FakeTensor)
    eng.n_envs, eng.nq, eng.device, eng.h, eng.launches = 4, 18, "cuda:0", None, 0
    eng.lib = types.SimpleNamespace(locosim_inverse=lambda h, a, b, s: calls.append((a, b)) or 0)
    eng._stream = lambda: None
    monkeypatch.setattr(engine_mod, "_ptr", lambda t: None if t is None else id(t))
    nb = 4 * 18 * 4
    qacc, out = _FakeTensor((4, 18), ptr=1 << 20), _FakeTensor((4, 18), ptr=(1 << 20) + nb)
    assert eng.inverse(qacc, out) is out and calls == [(id(qacc), id(out))]
    bad_inputs = [_FakeTensor((4, 17)), _FakeTensor((3, 18)), _FakeTensor((4, 18, 1)), _FakeTensor((4, 18), "float64"),
                  _FakeTensor((4, 18), contiguous=False), _FakeTensor((4, 18), device="cuda:1"), np.zeros((4, 18), np.float32)]
    for bad in bad_inputs:
        with pytest.raises(ValueError):
            eng.inverse(bad, out)
        with pytest.raises(ValueError):
            eng.inverse(qacc, bad)
    for off in (0, nb - 4, -(nb - 4)):                          # overlapping buffers are refused
        with pytest.raises(ValueError):
            eng.inverse(qacc, _FakeTensor((4, 18), ptr=(1 << 20) + off))
    assert len(calls) == 1


def test_dof_index(bundled_only):
    env = make_task("UnitreeA1.simple")
    names = list(env._model.jnt_names)
    assert [env.dof_index(n) for n in names] == list(range(env._model.nv))
    with pytest.raises(ValueError, match="no joint"):
        env.dof_index("not_a_joint")


def test_4ages_all_refuses_inverse_dynamics(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    env = LocoEnv.make("HumanoidTorque4Ages.walk.all.real", num_envs=8, debug=True)
    for call in (lambda: env.inverse_dynamics(None), env.create_dataset_inverse, lambda: env.dof_index("pelvis_tx")):
        with pytest.raises(NotImplementedError):
            call()


def test_dataset_rows_and_acceleration_on_the_serial_core(emu, ref, bundled_only):
    """Row r of create_dataset_inverse: (traj, sample) -> (traj, sample + 1), the reset state of (traj, sample) at
    qacc = (qvel[sample + 1] - qvel[sample]) * float32(1 / (timestep * n_substeps)); here on the serial core and the
    reference for a few rows of the dataset's order"""
    from loco_mujoco_b200 import modelpack
    env = make_task("UnitreeA1.simple")
    spec, m = env.task_spec(), env._model
    mb, tb = blobs(env)
    nv, n_traj, traj_len = m.nv, spec.table.shape[0], spec.table.shape[1]
    inv_dt = np.float32(1.0 / (float(np.float32(m.opt_timestep)) * spec.n_substeps))
    s = _emu(emu, modelpack.pack(m))
    sim = ivr.InverseSim(ref, mb, tb, geom_type=m.geom_type)
    per = traj_len - 1
    for r in (0, per - 1, n_traj * per - 1):
        tj, sp = divmod(r, per)
        row0, row1 = spec.table[tj, sp].astype(np.float32), spec.table[tj, sp + 1].astype(np.float32)
        q = row0[:nv].copy()
        q[list(spec.recenter)] = 0.0
        v0, v1 = row0[nv:2 * nv], row1[nv:2 * nv]
        qacc = (v1 - v0) * inv_dt                                # float32 arithmetic, as the kernel
        got = _emu_inverse(emu, s, q, v0, qacc)
        want = sim.at(q.astype(np.float64), v0.astype(np.float64), qacc.astype(np.float64))
        ok, ratio = ivr.within(got, want["qfrc"], want["scale"])
        assert ok or sim.explained(q.astype(np.float64), v0.astype(np.float64), qacc.astype(np.float64), got, want["qfrc"]), \
            (r, ratio)
    sim.close()
    emu.emu_destroy(s)
