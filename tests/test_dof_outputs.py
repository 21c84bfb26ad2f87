"""Per-dof outputs (MuJoCo's qfrc_actuator / qfrc_constraint / qacc, include/locosim.h locosim_set_dof_outputs) without a GPU:
the serial build of the CUDA core against the fp64 reference (tests/dof_outputs_ref.py), and the host-side rules. The
physics that pins the meaning of the three components on the reference (analytic actuator clamps, the joint-space balance
M qacc = qfrc_smooth + qfrc_constraint, a joint limit) is in tests/test_position_control.py."""
import types

import numpy as np
import pytest

import dof_outputs_ref as dor
from full_body import make_variant
from helpers import blobs
from position_mode import Sim, compile_xml, make_position

# Tolerance of the serial core (fp32) against the fp64 reference, per component: 1e-4 of the largest magnitude of that
# component over the dofs of the state (at least 1e-4 in its unit). The three components carry the relative error of an fp32
# forward evaluation and of a control step's fp32 drift from the fp64 trajectory (4-25 sub-steps); measured on the serial
# build from reset-table states under random actions: at most 1.2e-6 (qfrc_actuator), 3.6e-6 (qfrc_constraint) and 1e-5
# (qacc) of the magnitude. Where a contact switches on or off within the step the oracle's own result jumps under an
# fp32-sized perturbation of the start state; there the error must stay within 10x that jump.
REL = 1e-4

TASKS = ["UnitreeA1.simple", "UnitreeA1.simple+position", "HumanoidTorque.run", "Talos.walk", "Atlas.walk+arms"]


@pytest.fixture(scope="module")
def ref():
    return dor.load()


def make_task(task, **kw):
    """make_variant for the task names above ("UnitreeA1.<task>+position": action_mode "position")"""
    if task.endswith("+position"):
        return make_position(task[:-len("+position")], **kw)
    return make_variant(task, **kw)


def within(got, want, gap=None):
    """per component: |got - want| <= REL * max(1, max |want|), or < 10x the oracle's own jump `gap` [3]"""
    err = np.abs(got - want).max(axis=0)
    tol = REL * np.maximum(1.0, np.abs(want).max(axis=0))
    if gap is None:
        return bool(np.all(err <= tol)), err, tol
    return bool(np.all((err <= tol) | (err < 10 * gap))), err, tol


@pytest.mark.parametrize("task", TASKS)
def test_serial_core_matches_the_reference(emu, ref, bundled_only, task):
    """The serial build of the CUDA core (same source as the kernels) for one control step from reset-table states under
    random actions, against the fp64 reference's sub-step mean"""
    from loco_mujoco_b200 import modelpack
    dor.emu_bind(emu)
    env = make_task(task)
    m, spec = env._model, env.task_spec()
    mb, tb = blobs(env)
    ints, reals = [np.ascontiguousarray(x) for x in modelpack.pack(m)]
    ints, reals = ints.astype(np.int32), reals.astype(np.float64)
    p = dor._p
    sim = emu.emu_create(p(ints), len(ints), p(reals), len(reals))
    assert sim
    out = np.zeros((m.nv, dor.DOF_DIM), dtype=np.float32)
    emu.emu_set_dof(sim, p(out))
    rng = np.random.RandomState(11)
    table = spec.table.reshape(-1, spec.table.shape[-1])
    user = env._model_user_features[0]
    allowed, constrained = 0, 0
    for i in rng.randint(len(table), size=8):
        oe = ref.env(mb, tb)
        oe.set_user(user)
        oe.reset_to(i // spec.table.shape[1], i % spec.table.shape[1])
        q, v = oe.get_state()
        a = rng.uniform(-1, 1, m.nu)
        ctrl = np.zeros(m.nu)
        ctrl[spec.act_idx] = a * spec.act_delta + spec.act_mean
        out[:] = np.nan
        emu.emu_reset(sim, p(np.ascontiguousarray(q)), p(np.ascontiguousarray(v)))
        emu.emu_set_ws(sim, p(np.zeros(m.nv)))
        emu.emu_step(sim, p(ctrl), spec.n_substeps)
        want, _, _ = dor.env_step(ref, oe, a)
        oe.close()
        constrained += int(np.abs(want[:, 1]).max() > 1.0)
        ok, err, tol = within(out, want)
        if not ok:
            gap = dor.sensitivity(ref, mb, tb, q, v, a, want, eps=1e-6, n_probe=8, user=user)
            ok, err, tol = within(out, want, gap)
            assert ok, (task, i, err, tol, gap)
            allowed += 1
    emu.emu_destroy(sim)
    assert constrained >= 4, "too few states with constraint forces"
    assert allowed <= 2, allowed


def test_serial_core_on_a_position_hinge(emu, ref):
    """the serial core on the hand-built pendulum of test_position_control: the actuator clamp, a joint limit, Euler with
    joint damping (qacc is the constrained acceleration, not the implicit-damping solve)"""
    from test_position_control import _hinge
    dor.emu_bind(emu)
    p = dor._p
    _, packed = compile_xml(_hinge(kp=10.0, force="-6 6", rng=' limited="true" range="-0.4 0.4"'))
    ints, reals = [np.ascontiguousarray(x) for x in packed]
    ints, reals = ints.astype(np.int32), reals.astype(np.float64)
    es = emu.emu_create(p(ints), len(ints), p(reals), len(reals))
    assert es
    out = np.full((1, dor.DOF_DIM), np.nan, dtype=np.float32)
    emu.emu_set_dof(es, p(out))
    sim = Sim(ref, packed)
    for q0, v0, c in ((0.0, 0.0, 0.3), (0.35, 2.0, 2.5), (-0.39, -1.0, -2.0)):
        emu.emu_reset(es, p(np.array([q0])), p(np.array([v0])))
        emu.emu_set_ws(es, p(np.zeros(1)))
        emu.emu_step(es, p(np.array([c])), 10)
        sim.reset([q0], [v0])
        want = dor.step(ref, sim.sim, [c], 10)
        assert np.abs(out - want).max() < 1e-4 * max(1.0, np.abs(want).max()), (q0, v0, c, out, want)
    assert out[0, 1] != 0.0                                      # the last case runs into the lower limit
    emu.emu_destroy(es)
    sim.close()


def test_registering_changes_nothing_else_in_the_serial_core(emu, bundled_only):
    """the same control steps with and without the outputs registered: identical state bits"""
    from loco_mujoco_b200 import modelpack
    dor.emu_bind(emu)
    p = dor._p
    for task in ("UnitreeA1.simple+position", "HumanoidTorque.run"):
        env = make_task(task)
        m, spec = env._model, env.task_spec()
        ints, reals = [np.ascontiguousarray(x) for x in modelpack.pack(m)]
        ints, reals = ints.astype(np.int32), reals.astype(np.float64)
        table = spec.table.reshape(-1, spec.table.shape[-1])
        rng = np.random.RandomState(5)
        ctrls = [np.ascontiguousarray(rng.uniform(-1, 1, m.nu) * spec.act_delta + spec.act_mean) for _ in range(3)]
        states = []
        for register in (False, True):
            es = emu.emu_create(p(ints), len(ints), p(reals), len(reals))
            out = np.zeros((m.nv, dor.DOF_DIM), dtype=np.float32)
            if register:
                emu.emu_set_dof(es, p(out))
            emu.emu_reset(es, p(np.ascontiguousarray(table[3, :m.nv])), p(np.ascontiguousarray(table[3, m.nv:2 * m.nv])))
            for c in ctrls:
                emu.emu_step(es, p(c), spec.n_substeps)
            q, v = np.zeros(m.nv), np.zeros(m.nv)
            emu.emu_get_state(es, p(q), p(v))
            states.append(np.concatenate([q, v]))
            emu.emu_destroy(es)
        assert np.array_equal(states[0], states[1]), task


# ---------------------------------------------------------------------------------------------------------------------
# host logic
# ---------------------------------------------------------------------------------------------------------------------
class _FakeTensor:
    def __init__(self, shape, dtype="float32", contiguous=True, device="cuda:0"):
        self.shape, self.dtype, self._c, self.device = shape, dtype, contiguous, device

    def is_contiguous(self):
        return self._c


def test_set_dof_outputs_validates_its_arguments(monkeypatch):
    """dtype / shape / layout / device checks happen before the engine is called (no device needed)"""
    from loco_mujoco_b200 import engine as engine_mod
    calls = []
    eng = object.__new__(engine_mod.CudaEngine)
    eng.torch = types.SimpleNamespace(float32="float32")
    eng.n_envs, eng.nq, eng.device, eng.h = 4, 18, "cuda:0", None
    eng.lib = types.SimpleNamespace(locosim_set_dof_outputs=lambda h, d: calls.append(d) or 0)
    monkeypatch.setattr(engine_mod, "_ptr", lambda t: None if t is None else id(t))
    ok = _FakeTensor((4, 18, 3))
    eng.set_dof_outputs(ok)
    eng.set_dof_outputs()
    assert calls == [id(ok), None] and eng._dof_out is None
    for bad in (_FakeTensor((4, 18, 6)), _FakeTensor((4, 17, 3)), _FakeTensor((3, 18, 3)), _FakeTensor((4, 18, 3), "float64"),
                _FakeTensor((4, 18, 3), contiguous=False), _FakeTensor((4, 18, 3), device="cuda:1")):
        with pytest.raises(ValueError):
            eng.set_dof_outputs(bad)
    assert len(calls) == 2
    assert engine_mod.DOF_DIM == 3


class _RecordingEngine:
    """Stands in for CudaEngine on a CPU-only box: records what the env registers."""

    def __init__(self, model_blobs, task_blobs, n_envs, device=0, **kw):
        import torch
        self.device, self.n_envs, self.calls = torch.device("cpu"), n_envs, []

    def set_dof_outputs(self, dof=None):
        self.calls.append(dof)

    def set_param_pool(self, pool):
        pass

    def close(self):
        pass


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "UnitreeA1.simple+position"])
def test_dof_outputs_are_lazy_and_survive_an_engine_rebuild(bundled_only, monkeypatch, task):
    from loco_mujoco_b200 import engine as engine_mod
    monkeypatch.setattr(engine_mod, "CudaEngine", _RecordingEngine)
    env = make_task(task, num_envs=5)
    eng = env._get_engine()
    assert eng.calls == []                                       # nothing registered until the tensor is asked for
    d = env.dof_outputs
    assert tuple(d.shape) == (5, env._model.nq, 3) and str(d.dtype) == "torch.float32" and d.is_contiguous()
    assert env._model.nq == env._model.nv == 18
    assert float(d.abs().max()) == 0.0                           # allocated zeroed
    assert eng.calls == [d] and env.dof_outputs is d and len(eng.calls) == 1
    env.set_launch_geometry(4)                                   # rebuilds the engine: the same tensor is registered again
    eng2 = env._get_engine()
    assert eng2 is not eng and eng2.calls == [d]


def test_4ages_all_refuses_dof_outputs(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    env = LocoEnv.make("HumanoidTorque4Ages.walk.all.real", num_envs=8, debug=True)
    with pytest.raises(NotImplementedError):
        env.dof_outputs
