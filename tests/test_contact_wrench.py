"""Contact outputs (MuJoCo's mj_contactForce summed per body, include/locosim.h locosim_set_contact_outputs) without a GPU: the
fp64 reference (tests/contact_wrench_ref.py) against hand-built scenes and physical laws, the serial build of the CUDA core
against that reference, and the host-side rules."""
import os
import tempfile
import types

import numpy as np
import pytest

import contact_wrench_ref as cwr
from full_body import make_variant
from helpers import blobs, make_env

# Tolerance of the serial core (fp32) against the fp64 reference, per wrench component: 2 N on forces, 2 N m on torques. This
# is the tolerance test_foot_forces_match_oracle accepts for the same forces (2e-3 of an observation scaled by 1 / 1000).
TOL = 2.0


@pytest.fixture(scope="module")
def ref():
    return cwr.load()


def _compile(xml):
    from loco_mujoco_b200 import mjcf, modelpack
    with tempfile.NamedTemporaryFile("w", suffix=".xml", delete=False) as f:
        f.write(xml)
        path = f.name
    try:
        m = mjcf.compile_model(mjcf.XmlHandle(path), fuse_static=False)
    finally:
        os.unlink(path)
    return m, modelpack.pack(m)


class _Sim:
    """a bare oracle sim of a compiled model"""

    def __init__(self, o, packed):
        import ctypes
        self.lib = o.lib
        self._keep = [np.ascontiguousarray(packed[0], dtype=np.int32), np.ascontiguousarray(packed[1], dtype=np.float64)]
        a, b = self._keep
        self.sim = ctypes.c_void_p(self.lib.ref_create(cwr._p(a), len(a), cwr._p(b), len(b)))
        assert self.sim.value
        self.o = o

    def reset(self, q, v):
        q, v = np.ascontiguousarray(q, dtype=np.float64), np.ascontiguousarray(v, dtype=np.float64)
        self.lib.ref_reset(self.sim, cwr._p(q), cwr._p(v))

    def state(self):
        q, v = np.zeros(self.lib.ref_nv(self.sim)), np.zeros(self.lib.ref_nv(self.sim))
        self.lib.ref_get_state(self.sim, cwr._p(q), cwr._p(v))
        return q, v

    def close(self):
        self.lib.ref_destroy(self.sim)


# A box resting on the floor, its geom off-centre in its body (the body can only translate: by symmetry its four corner
# contacts then carry equal forces, and the torque about the body origin is (geom centre - xpos) x weight).
BOX_XML = """
<mujoco model="box">
  <option timestep="0.002" integrator="Euler" cone="pyramidal"/>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 1" condim="3"/>
    <body name="box" pos="0 0 0.2">
      <joint name="x" type="slide" axis="1 0 0"/><joint name="y" type="slide" axis="0 1 0"/>
      <joint name="z" type="slide" axis="0 0 1"/>
      <geom name="g" type="box" size="0.1 0.08 0.05" pos="0.3 -0.2 -0.15" mass="4" condim="3"/>
    </body>
  </worldbody>
</mujoco>
"""
# A sphere on an elliptic cone with torsional and rolling friction (condim 6), free to spin about the vertical
SPIN_XML = """
<mujoco model="spin">
  <option timestep="0.002" integrator="Euler" cone="elliptic"/>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 1" condim="6" friction="1 0.05 0.001"/>
    <body name="ball" pos="0 0 0.1">
      <joint name="z" type="slide" axis="0 0 1"/><joint name="spin" type="hinge" axis="0 0 1"/>
      <geom name="g" type="sphere" size="0.1" mass="2" condim="6" friction="1 0.05 0.001"/>
    </body>
  </worldbody>
</mujoco>
"""


def _settle(sim, nv, q0, n=400):
    sim.reset(q0, np.zeros(nv))
    for _ in range(n):
        sim.lib.ref_step(sim.sim, None, 1)
    return sim.state()


def test_box_at_rest_off_centre(ref):
    m, packed = _compile(BOX_XML)
    sim = _Sim(ref, packed)
    q, v = _settle(sim, m.nv, np.zeros(3))
    assert np.abs(v).max() < 1e-6
    w = cwr.step(ref, sim.sim, np.zeros(0), 5)
    W = 4 * 9.81
    assert np.array_equal(w[0], np.zeros(6))                                # the world row
    assert np.allclose(w[1, :3], [0, 0, W], rtol=0, atol=1e-6 * W), w[1]
    xpos = np.array([q[0], q[1], 0.2 + q[2]])
    centre = xpos + [0.3, -0.2, -0.15]
    want = np.cross(centre - xpos, [0, 0, W])                               # (0.2 W, 0.3 W, 0): analytic r x F
    assert np.allclose(w[1, 3:], want, rtol=0, atol=1e-6 * W), (w[1, 3:], want)
    # the four corners, each a quarter of the weight at its own lever arm, sum to the same torque
    cons = cwr.contacts(ref, sim.sim)
    assert len(cons) == 4 and np.allclose(cons[:, 16], W / 4, rtol=1e-6)
    sim.close()


def test_spinning_sphere_torsion_opposes_the_spin(ref):
    m, packed = _compile(SPIN_XML)
    sim = _Sim(ref, packed)
    q, _ = _settle(sim, m.nv, np.zeros(2))
    W = 2 * 9.81
    for spin in (1.0, -1.0):          # (a faster spin makes the soft elliptic cone lift the ball off the floor)
        sim.reset(q, [0.0, spin])
        w = cwr.step(ref, sim.sim, np.zeros(0), 5)
        cons = cwr.contacts(ref, sim.sim)
        assert len(cons) == 1 and cons[0, 15] == 6
        assert np.array_equal(cons[0, 4:7], [0, 0, 1]) and cons[0, 13] == 0      # floor = geom1: n points up, into the ball
        assert np.allclose(w[1, :3], [0, 0, W], rtol=0.01, atol=1e-3), w[1]
        tz = w[1, 5]
        # the torsional component acts against the spin, bounded by torsional friction x normal force
        assert np.sign(tz) == -np.sign(spin) and 0.01 * W * 0.05 < abs(tz) <= 1.01 * 0.05 * W, (spin, tz)
        assert abs(w[1, 3]) < 1e-6 and abs(w[1, 4]) < 1e-6
        assert np.array_equal(w[0], np.zeros(6))
    sim.close()


def test_serial_core_on_the_hand_built_scenes(emu, ref):
    """the serial CUDA core on both scenes: the elliptic condim-6 decode (torsion included) and the pyramidal one"""
    cwr.emu_bind(emu)
    p = cwr._p
    for xml, q0, v1 in ((BOX_XML, np.zeros(3), np.array([0.3, -0.2, 0.0])), (SPIN_XML, np.zeros(2), np.array([0.0, 1.0]))):
        m, packed = _compile(xml)
        sim = _Sim(ref, packed)
        q, _ = _settle(sim, m.nv, q0)
        ints, reals = [np.ascontiguousarray(x) for x in packed]
        ints, reals = ints.astype(np.int32), reals.astype(np.float64)
        es = emu.emu_create(p(ints), len(ints), p(reals), len(reals))
        assert es
        out = np.full((m.nbody, 6), np.nan, dtype=np.float32)
        emu.emu_set_contact(es, p(out))
        q = np.ascontiguousarray(q)
        emu.emu_reset(es, p(q), p(v1))
        emu.emu_step(es, p(np.zeros(1)), 5)
        sim.reset(q, v1)
        want = cwr.step(ref, sim.sim, np.zeros(0), 5)
        assert np.array_equal(out[0], np.zeros(6))
        assert np.abs(out - want).max() < 1e-3 * max(1.0, np.abs(want).max()), (out, want)
        emu.emu_destroy(es)
        sim.close()


def test_at_rest_weight_and_foot_forces(ref, bundled_only):
    """the settle set-up of test_foot_forces: the body forces carry the weight, and A1's foot rows have the normal force of
    the foot-force observation (the same mj_contactForce decode, the same sub-step mean)"""
    env = make_env("UnitreeA1.simple", use_foot_forces=True, use_absorbing_states=False)
    spec, m = env.task_spec(), env._model
    n_grf = spec.n_grf
    mb, tb = blobs(env)
    oe = ref.env(mb, tb)
    oe.reset_to(0, 10)
    zero = np.zeros(env.info.action_space.shape[0])
    for _ in range(250):
        oe.step(zero)
    q, v = oe.get_state()
    ws = np.zeros(m.nv)
    ref.lib.ref_get_warmstart(oe.sim, cwr._p(ws))
    assert np.abs(v).max() < 5e-2, "not at rest"
    w, _, _ = cwr.env_step(ref, oe, zero)
    weight = m.body_mass.sum() * 9.81
    total = w[:, :3].sum(axis=0)
    assert abs(total[2] - weight) < 0.01 * weight and np.abs(total[:2]).max() < 0.01 * weight, (total, weight)
    # the same step through the observation
    o2 = ref.env(mb, tb)
    o2.set_state(q, v, ws)
    obs, _, _ = o2.step(zero)
    grf = obs[-3 * n_grf:].reshape(n_grf, 3) * 1000.0
    # and sub-step by sub-step: a foot body's row less its other floor contacts (A1 lies on its calves) is its foot contact
    o3 = ref.env(mb, tb)
    o3.set_state(q, v, ws)
    ctrl = np.zeros(m.nu)
    ctrl[spec.act_idx] = spec.act_mean
    feet = np.zeros(n_grf)
    mean = np.zeros_like(w)
    for _ in range(spec.n_substeps):
        ws_k = cwr.step(ref, o3.sim, ctrl, 1)
        mean += ws_k / spec.n_substeps
        cons = cwr.contacts(ref, o3.sim)
        for g in range(n_grf):
            b = {int(m.geom_bodyid[i]) for i in range(m.ngeom) if spec.grf_group[i] == g}
            assert len(b) == 1
            b = b.pop()
            others = [c for c in cons if m.geom_bodyid[int(c[14])] == b and spec.grf_group[int(c[14])] != g]
            assert all(c[13] == 0 and np.array_equal(c[4:7], [0, 0, 1]) for c in others)       # floor contacts, normal up
            feet[g] += (ws_k[b, 2] - sum(c[16] for c in others)) / spec.n_substeps
    assert np.allclose(mean, w, rtol=0, atol=1e-9 * np.abs(w).max())      # env_step's row is the sub-step mean
    assert np.all(grf[:, 0] > 0.1)
    assert np.allclose(feet, grf[:, 0], rtol=1e-6, atol=1e-9), (feet, grf[:, 0])
    oe.close()
    o2.close()
    o3.close()


def test_newton_third_law_in_self_contacts(ref, bundled_only):
    """HumanoidTorque states with bone-bone contacts (reset-table poses with the joints bent at random until bones
    interpenetrate): without the floor contacts, the body rows sum to a zero force and to a zero torque about the origin (each
    self contact appears twice with opposite signs)"""
    env = make_env("HumanoidTorque.run")
    m, spec = env._model, env.task_spec()
    mb, tb = blobs(env)
    oe = ref.env(mb, tb)
    table = spec.table.reshape(-1, spec.table.shape[-1])
    rng = np.random.RandomState(3)
    found = 0
    for i in rng.randint(len(table), size=100):
        q, v = table[i, :m.nv].copy(), table[i, m.nv:2 * m.nv]
        q[6:] += rng.uniform(-1.2, 1.2, m.nv - 6)               # (dofs 0-5: the root)
        oe.set_state(q, v)
        ref.lib.ref_forward(oe.sim, None)
        cons = cwr.contacts(ref, oe.sim)
        b1, b2 = m.geom_bodyid[cons[:, 13].astype(int)], m.geom_bodyid[cons[:, 14].astype(int)]
        self_c = (b1 > 0) & (b2 > 0)
        if not self_c.any() or np.abs(cons[self_c, 16:]).max() == 0:
            continue
        w = cwr.wrench_now(ref, oe.sim)
        xpos, xquat = np.zeros((m.nbody, 3)), np.zeros((m.nbody, 4))
        ref.lib.ref_get_frames(oe.sim, cwr._p(xpos), cwr._p(xquat))
        F, T = w[:, :3].sum(axis=0), (w[:, 3:] + np.cross(xpos, w[:, :3])).sum(axis=0)
        for c, bb1, bb2 in zip(cons, b1, b2):                # take the floor contacts out
            if bb1 > 0 and bb2 > 0:
                continue
            f = c[16:]
            n, t1, t2 = c[4:7], c[7:10], c[10:13]
            Fw, Tw = f[0] * n + f[1] * t1 + f[2] * t2, f[3] * n + f[4] * t1 + f[5] * t2
            s = 1.0 if bb2 > 0 else -1.0
            F -= s * Fw
            T -= s * (Tw + np.cross(c[1:4], Fw))
        scale = np.abs(w).max() * (1 + np.abs(xpos).max())
        assert np.abs(F).max() < 1e-12 * scale and np.abs(T).max() < 1e-12 * scale, (F, T, scale)
        found += 1
        if found == 5:
            break
    assert found >= 3, "no states with bone-bone contact forces"
    oe.close()


TASKS = ["UnitreeA1.simple", "HumanoidTorque.run", "Talos.walk", "Atlas.walk+arms+back", "Talos.walk+arms"]


@pytest.mark.parametrize("task", TASKS)
def test_serial_core_matches_the_reference(emu, ref, bundled_only, task):
    """The serial build of the CUDA core (same source as the kernels) for one control step from reset-table states under
    random actions, against the fp64 reference's sub-step mean, within TOL; where the oracle's own result jumps under an
    fp32-sized perturbation of the start state (a contact switching within the step), within 10x that jump."""
    from loco_mujoco_b200 import modelpack
    cwr.emu_bind(emu)
    env = make_variant(task)
    m, spec = env._model, env.task_spec()
    assert m.nbody <= 32
    mb, tb = blobs(env)
    ints, reals = [np.ascontiguousarray(x) for x in modelpack.pack(m)]
    ints, reals = ints.astype(np.int32), reals.astype(np.float64)
    p = cwr._p
    sim = emu.emu_create(p(ints), len(ints), p(reals), len(reals))
    assert sim
    out = np.zeros((m.nbody, 6), dtype=np.float32)
    emu.emu_set_contact(sim, p(out))
    rng = np.random.RandomState(11)
    table = spec.table.reshape(-1, spec.table.shape[-1])
    user = env._model_user_features[0]
    worst, touched, allowed = 0.0, 0, 0
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
        want, _, _ = cwr.env_step(ref, oe, a)
        oe.close()
        assert np.array_equal(out[0], np.zeros(6))
        err = float(np.abs(out - want).max())
        touched += int(np.abs(want).max() > 1.0)
        if err > TOL:
            gap = cwr.sensitivity(ref, mb, tb, q, v, a, want, eps=1e-6, n_probe=8, user=user)
            assert err < 10 * gap, (task, i, err, gap)
            allowed += 1
        else:
            worst = max(worst, err)
    emu.emu_destroy(sim)
    assert touched >= 4, "too few states with contact forces"
    assert allowed <= 2, allowed


# ---------------------------------------------------------------------------------------------------------------------
# host logic
# ---------------------------------------------------------------------------------------------------------------------
class _FakeTensor:
    def __init__(self, shape, dtype="float32", contiguous=True, device="cuda:0"):
        self.shape, self.dtype, self._c, self.device = shape, dtype, contiguous, device

    def is_contiguous(self):
        return self._c


def test_set_contact_outputs_validates_its_arguments(monkeypatch):
    """dtype / shape / layout / device checks happen before the engine is called (no device needed)"""
    from loco_mujoco_b200 import engine as engine_mod
    calls = []
    eng = object.__new__(engine_mod.CudaEngine)
    eng.torch = types.SimpleNamespace(float32="float32")
    eng.n_envs, eng.nbody, eng.device, eng.h = 4, 3, "cuda:0", None
    eng.lib = types.SimpleNamespace(locosim_set_contact_outputs=lambda h, c: calls.append(c) or 0)
    monkeypatch.setattr(engine_mod, "_ptr", lambda t: None if t is None else id(t))
    ok = _FakeTensor((4, 3, 6))
    eng.set_contact_outputs(ok)
    eng.set_contact_outputs()
    assert calls == [id(ok), None] and eng._contact_out is None
    for bad in (_FakeTensor((4, 3, 13)), _FakeTensor((4, 4, 6)), _FakeTensor((3, 3, 6)), _FakeTensor((4, 3, 6), "float64"),
                _FakeTensor((4, 3, 6), contiguous=False), _FakeTensor((4, 3, 6), device="cuda:1")):
        with pytest.raises(ValueError):
            eng.set_contact_outputs(bad)
    assert len(calls) == 2
    assert engine_mod.CONTACT_DIM == 6


class _RecordingEngine:
    """Stands in for CudaEngine on a CPU-only box: records what the env registers."""
    made = []

    def __init__(self, model_blobs, task_blobs, n_envs, device=0, **kw):
        import torch
        self.device, self.n_envs, self.calls = torch.device("cpu"), n_envs, []
        _RecordingEngine.made.append(self)

    def set_contact_outputs(self, contact=None):
        self.calls.append(contact)

    def set_param_pool(self, pool):
        pass

    def close(self):
        pass


def test_contact_wrench_is_lazy_and_survives_an_engine_rebuild(bundled_only, monkeypatch):
    from loco_mujoco_b200 import engine as engine_mod
    monkeypatch.setattr(engine_mod, "CudaEngine", _RecordingEngine)
    env = make_env("UnitreeA1.simple", num_envs=5)
    eng = env._get_engine()
    assert eng.calls == []                                       # nothing registered until the tensor is asked for
    c = env.contact_wrench
    assert tuple(c.shape) == (5, env._model.nbody, 6) and str(c.dtype) == "torch.float32" and c.is_contiguous()
    assert float(c.abs().max()) == 0.0                           # allocated zeroed
    assert eng.calls == [c] and env.contact_wrench is c and len(eng.calls) == 1
    env.set_launch_geometry(4)                                   # rebuilds the engine: the same tensor is registered again
    eng2 = env._get_engine()
    assert eng2 is not eng and eng2.calls == [c]


def test_4ages_all_refuses_contact_outputs(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    env = LocoEnv.make("HumanoidTorque4Ages.walk.all.real", num_envs=8, debug=True)
    with pytest.raises(NotImplementedError):
        env.contact_wrench
