"""Forward dynamics under an action (MuJoCo 2.3.7's mj_forward + mj_rnePostConstraint, include/locosim.h locosim_forward)
without a GPU: the fp64 reference (tests/forward_ref.py) on hand-built scenes with closed-form answers and against
identities of rigid-body mechanics for every bundled model, the serial build of the CUDA core against that reference for
every kernel configuration, and the host-side rules."""
import types

import numpy as np
import pytest

import forward_ref as fwr
from full_body import make_variant
from helpers import blobs
from position_mode import compile_xml, make_position

G = 9.81
# one task per kernel configuration (locosim_host.h select_cfg)
CFG_TASKS = {"CfgEllEuler": "UnitreeA1.simple", "CfgPyrEuler": "Talos.walk", "CfgPyrRK4": "HumanoidTorque.run",
             "CfgPyrEuler29": "UnitreeH1.walk+arms", "CfgPyrRK4_31": "Atlas.walk+arms", "CfgPyrEuler31": "Talos.walk+arms"}
# every bundled model: the configurations' tasks, UnitreeA1 under position control, the models without arms, the four
# HumanoidTorque4Ages humanoids and the carry tasks (their first carried weight)
IDENTITY_TASKS = list(CFG_TASKS.values()) + ["UnitreeA1.simple+position", "UnitreeG1.walk", "Atlas.walk", "UnitreeH1.walk",
                                             "HumanoidTorque4Ages.walk.1", "HumanoidTorque4Ages.walk.2",
                                             "HumanoidTorque4Ages.walk.3", "HumanoidTorque4Ages.walk.4", "Atlas.carry",
                                             "Talos.carry", "UnitreeH1.carry"]


@pytest.fixture(scope="module")
def ref():
    return fwr.load()


def make_task(task, **kw):
    """make_variant for the task names above ("UnitreeA1.<task>+position": action_mode "position")"""
    if task.endswith("+position"):
        return make_position(task[:-len("+position")], **kw)
    return make_variant(task, **kw)


def _emu(emu, packed):
    fwr.emu_bind(emu)
    ints, reals = [np.ascontiguousarray(x) for x in packed]
    ints, reals = ints.astype(np.int32), reals.astype(np.float64)
    s = emu.emu_create(fwr._p(ints), len(ints), fwr._p(reals), len(reals))
    assert s
    return s


def _ctrl(spec, a):
    c = np.zeros(len(spec.act_idx))
    c[spec.act_idx] = a * spec.act_delta + spec.act_mean
    return c


def _states(env, ref, n, seed):
    """n states of the fp64 reference: reset-table rows advanced by two control steps under random actions (contacts
    active, velocities off the mocap clip)"""
    spec = env.task_spec()
    mb, tb = blobs(env)
    rng = np.random.RandomState(seed)
    out = []
    for i in rng.randint(spec.table.shape[0] * spec.table.shape[1], size=n):
        oe = ref.env(mb, tb)
        oe.set_user(env._model_user_features[0])
        oe.reset_to(i // spec.table.shape[1], i % spec.table.shape[1])
        for _ in range(2):
            oe.step(rng.uniform(-1, 1, env._model.nu))
        out.append(oe.get_state())
        oe.close()
    return out


# ---------------------------------------------------------------------------------------------------------------------
# closed-form scenes
# ---------------------------------------------------------------------------------------------------------------------
# a pendulum on a hinge about x with its centre of mass off the axis in x: gravity's moment about the hinge axis is 0, so
# it rests; the joint carries the weight and the moment about y
PENDULUM_XML = """
<mujoco model="pendulum">
  <option timestep="0.002" integrator="Euler"/>
  <worldbody>
    <body name="bob" pos="0 0 1">
      <joint name="h" type="hinge" axis="1 0 0"/>
      <inertial pos="0.3 0 -0.5" mass="2" diaginertia="0.1 0.2 0.3"/>
      <geom name="g" type="sphere" size="0.05" contype="0" conaffinity="0"/>
    </body>
  </worldbody>
</mujoco>
"""
# a body on three slides (it cannot rotate), no floor: it falls freely
FALL_XML = """
<mujoco model="fall">
  <option timestep="0.002" integrator="Euler"/>
  <worldbody>
    <body name="b" pos="0 0 1">
      <joint name="x" type="slide" axis="1 0 0"/><joint name="y" type="slide" axis="0 1 0"/>
      <joint name="z" type="slide" axis="0 0 1"/>
      <inertial pos="0.1 -0.2 0.05" mass="3" diaginertia="0.1 0.1 0.1"/>
      <geom name="g" type="sphere" size="0.1" contype="0" conaffinity="0"/>
    </body>
  </worldbody>
</mujoco>
"""
# a planar two-link arm (hinges about y, links along x), no gravity, both joints driven by motors
ARM_XML = """
<mujoco model="arm">
  <compiler angle="radian"/>
  <option timestep="0.002" integrator="Euler" gravity="0 0 0"/>
  <worldbody>
    <body name="l1" pos="0 0 1">
      <joint name="j1" type="hinge" axis="0 1 0"/>
      <inertial pos="0.25 0 0" mass="1.5" diaginertia="0.01 0.04 0.04"/>
      <geom name="g1" type="sphere" size="0.02" contype="0" conaffinity="0"/>
      <body name="l2" pos="0.5 0 0">
        <joint name="j2" type="hinge" axis="0 1 0"/>
        <inertial pos="0.2 0 0" mass="0.8" diaginertia="0.005 0.02 0.02"/>
        <geom name="g2" type="sphere" size="0.02" contype="0" conaffinity="0"/>
      </body>
    </body>
  </worldbody>
  <actuator>
    <motor joint="j1" gear="1"/><motor joint="j2" gear="1"/>
  </actuator>
</mujoco>
"""
# a frictionless ball on three slides resting in the floor, default solref / solimp
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


def _scene(ref, emu, xml):
    m, packed = compile_xml(xml)
    return m, fwr.ForwardSim(ref, packed), _emu(emu, packed)


def _both(r, emu, s, m, q, v, ctrl=()):
    """(reference, serial core) outputs at (q, v, ctrl)"""
    want = r.forward(q, v, np.asarray(ctrl, dtype=np.float64) if len(ctrl) else None)
    got = fwr.emu_forward(emu, s, m.nv, m.nbody, q, v, np.asarray(ctrl, dtype=np.float64))
    return want, got


def test_a_resting_pendulum_hangs_on_its_joint(emu, ref):
    m, r, s = _scene(ref, emu, PENDULUM_XML)
    want, got = _both(r, emu, s, m, [0.0], [0.0])
    mg, arm = 2 * G, np.array([0.3, 0.0, -0.5])
    # the joint holds the weight and its moment about xpos: F = (0, 0, m g), T = arm x F
    wrench = np.concatenate([[0, 0, mg], np.cross(arm, [0, 0, mg])])
    for out, tol in ((want, 1e-12), (got, 1e-5)):
        assert np.allclose(out["dof"][0], 0.0, atol=tol * 10)
        assert np.allclose(out["cfrc_int"][1], wrench, rtol=0, atol=tol * mg)
        assert np.allclose(out["body_acc"][1], [0, 0, 0, 0, 0, G], rtol=0, atol=tol * G)      # an accelerometer at rest
        assert np.allclose(out["body_acc"][0], [0, 0, 0, 0, 0, G], rtol=0, atol=tol * G)      # row 0: (0, -gravity)
        assert not np.any(out["cfrc_ext"]) and not np.any(out["cfrc_int"][0])
    r.close()
    emu.emu_destroy(s)


def test_a_falling_body_reads_zero_acceleration(emu, ref):
    m, r, s = _scene(ref, emu, FALL_XML)
    for v in ([0, 0, 0], [1.5, -0.7, 2.0]):
        want, got = _both(r, emu, s, m, [0.2, -0.1, 0.4], v)
        for out, tol in ((want, 1e-12), (got, 1e-5)):
            assert np.allclose(out["dof"][:, 2], [0, 0, -G], atol=tol * G)
            assert np.allclose(out["body_acc"][1], 0.0, atol=tol * G)
            assert np.allclose(out["cfrc_int"][1], 0.0, atol=tol * 3 * G)
    r.close()
    emu.emu_destroy(s)


def test_a_two_link_arm_in_motion(emu, ref):
    """body_acc of the second link's origin = L1 (u'(q1) qacc1 - u(q1) qd1^2), u(q) = (cos q, 0, -sin q) (rotation about
    y), its angular acceleration qacc1 + qacc2; the joint force on the second link = m2 times its CoM acceleration"""
    m, r, s = _scene(ref, emu, ARM_XML)
    q, v, ctrl = np.array([0.4, -0.9]), np.array([1.3, -2.1]), np.array([0.7, -0.3])
    want, got = _both(r, emu, s, m, q, v, ctrl)

    def u(t):
        return np.array([np.cos(t), 0.0, -np.sin(t)])

    def du(t):
        return np.array([-np.sin(t), 0.0, -np.cos(t)])

    for out, tol in ((want, 1e-9), (got, 2e-5)):
        a = out["dof"][:, 2]
        assert np.allclose(out["dof"][:, 0], ctrl, atol=tol)
        acc2 = 0.5 * (du(q[0]) * a[0] - u(q[0]) * v[0] ** 2)
        t, td, tdd = q.sum(), v.sum(), a.sum()
        acc_com2 = acc2 + 0.2 * (du(t) * tdd - u(t) * td ** 2)
        acc_com1 = 0.25 * (du(q[0]) * a[0] - u(q[0]) * v[0] ** 2)
        scale = max(1.0, np.abs(acc2).max())
        assert np.allclose(out["body_acc"][2, 3:], acc2, atol=tol * scale), (out["body_acc"][2], acc2)
        assert np.allclose(out["body_acc"][2, :3], [0, tdd, 0], atol=tol * scale)
        assert np.allclose(out["body_acc"][1, :3], [0, a[0], 0], atol=tol * scale)
        assert np.allclose(out["cfrc_int"][2, :3], 0.8 * acc_com2, atol=tol * scale)
        # the base carries both links
        assert np.allclose(out["cfrc_int"][1, :3], 0.8 * acc_com2 + 1.5 * acc_com1, atol=tol * scale)
        # the second joint's motor torque is the y moment the first link exerts on the second
        assert abs(out["cfrc_int"][2, 4] - ctrl[1]) < tol * scale
    r.close()
    emu.emu_destroy(s)


def test_a_ball_resting_in_the_floor_is_held_by_its_contact(emu, ref):
    """soft contact at depth below solimp's width, qvel = 0: with D = 1 / R, aref = K imp depth, the solver's qacc_z =
    (D aref - m g) / (m + D), and the contact force m (qacc_z + g) is cfrc_ext; the slides carry nothing"""
    m, r, s = _scene(ref, emu, BALL_XML)
    depth, mass = 0.004, 3.0
    dmax, tc, dr = 0.95, 0.02, 1.0
    K = 1.0 / (dmax * dmax * tc * tc * dr * dr)
    imp, diag = dmax, float(m.geom_invweight0[1, 0])
    D = imp / ((1 - imp) * diag)
    aref = K * imp * depth
    az = (D * aref - mass * G) / (mass + D)
    f = mass * (az + G)
    want, got = _both(r, emu, s, m, [0.0, 0.0, 0.1 - depth], [0, 0, 0])
    for out, tol in ((want, 1e-9), (got, 1e-4)):
        assert abs(out["dof"][2, 2] - az) < tol * max(1.0, abs(az)), (out["dof"][:, 2], az)
        assert np.allclose(out["cfrc_ext"][1], [0, 0, f, 0, 0, 0], atol=tol * f)
        assert np.allclose(out["cfrc_int"][1], 0.0, atol=tol * f)
        assert np.allclose(out["body_acc"][1, 3:], [0, 0, az + G], atol=tol * f)
    assert 0.5 * mass * G < f < 2 * mass * G                       # of the order of the weight
    r.close()
    emu.emu_destroy(s)


# ---------------------------------------------------------------------------------------------------------------------
# identities of the fp64 reference for every bundled model
# ---------------------------------------------------------------------------------------------------------------------
def _chains(m):
    """chain[b] = the dofs on the path root..b; subtree[b] = b and its descendants"""
    nb = m.nbody
    parent = np.asarray(m.body_parentid)
    jb = np.asarray(m.jnt_bodyid)
    anc = [set() for _ in range(nb)]
    for b in range(1, nb):
        anc[b] = anc[parent[b]] | {b}
    chain = [[d for d in range(m.nv) if jb[d] in anc[b]] for b in range(nb)]
    subtree = [[c for c in range(nb) if b in anc[c]] for b in range(nb)]
    return chain, subtree, parent


def _jac(r, q, chain):
    """body Jacobians at xpos [nb, 6, nv] (angular rows, then linear) from cdof about the CoM"""
    xpos, cdof, com = r.kin(q)
    J = np.zeros((r.nb, 6, r.nv))
    for b in range(1, r.nb):
        for d in chain[b]:
            J[b, :3, d] = cdof[d, :3]
            J[b, 3:, d] = cdof[d, 3:] + np.cross(cdof[d, :3], xpos[b] - com[1])
    return J


@pytest.mark.parametrize("task", IDENTITY_TASKS)
def test_reference_identities(ref, bundled_only, task):
    """On the fp64 reference at states under random actions and applied forces:
    body_acc = J qacc + Jdot qvel - (0, g), Jdot qvel from central differences of J along qvel;
    Newton-Euler per body, cfrc_int[b] - sum over children of cfrc_int[c] + cfrc_ext[b] + m_b g = the rate of b's momentum
    (about xipos: m a_com and I alpha + w x I w);
    cdof_j . cfrc_int[body(j)] = qfrc_actuator + qfrc_passive + qfrc_applied + qfrc_constraint - its contact part
    - armature_j qacc_j (the rotor's inertia is the joint's own, not a body's)"""
    env = make_task(task)
    m, spec = env._model, env.task_spec()
    mb, tb = blobs(env)
    r = fwr.ForwardSim(ref, mb, tb, env._model_user_features[0])
    chain, subtree, parent = _chains(m)
    mass = np.asarray(m.body_mass, dtype=np.float64)
    grav = np.array([0.0, 0.0, -G])
    rng = np.random.RandomState(4)
    contacts = 0
    for q, v in _states(env, ref, 3, 5):
        qfrc = rng.normal(0, 5, m.nv)
        xfrc = rng.normal(0, 5, (m.nbody, 6))
        o = r.forward(q, v, _ctrl(spec, rng.uniform(-1, 1, m.nu)), xfrc=xfrc, qfrc=qfrc)
        qacc = o["dof"][:, 2]
        contacts += int(np.abs(o["cfrc_ext"]).max() > 0)
        # (a) body accelerations from the Jacobians
        h = 1e-6
        J = _jac(r, q, chain)
        Jd = (_jac(r, q + h * v, chain) - _jac(r, q - h * v, chain)) / (2 * h)
        acc = J @ qacc + Jd @ v
        acc[:, 3:] -= grav
        acc[0, 3:] = -grav
        scale = max(1.0, np.abs(acc).max())
        assert np.allclose(o["body_acc"], acc, rtol=0, atol=1e-5 * scale), (task, np.abs(o["body_acc"] - acc).max())
        # (b) Newton-Euler per body about xipos
        xpos, _, _ = r.kin(q)
        xipos, ci, com = o["xipos"], o["cinert"], o["subtree_com"][1]
        big = max(1.0, np.abs(o["cfrc_int"]).max())
        for b in range(1, m.nbody):
            w_b = J[b, :3] @ v
            a_p = o["body_acc"][b, 3:] + grav                          # true acceleration of xpos
            d = xipos[b] - xpos[b]
            a_com = a_p + np.cross(o["body_acc"][b, :3], d) + np.cross(w_b, np.cross(w_b, d))
            F = o["cfrc_int"][b, :3] + o["cfrc_ext"][b, :3] + mass[b] * grav
            T = o["cfrc_int"][b, 3:] + o["cfrc_ext"][b, 3:]
            for c in range(b + 1, m.nbody):
                if parent[c] == b:
                    F = F - o["cfrc_int"][c, :3]
                    T = T - o["cfrc_int"][c, 3:] - np.cross(xpos[c] - xpos[b], o["cfrc_int"][c, :3])
            # torques about xipos: T + (xpos - xipos) x (the forces through xpos); gravity acts at xipos
            T = T + np.cross(xpos[b] - xipos[b], F - mass[b] * grav)
            dc = xipos[b] - com
            Iw = np.array([[ci[b, 0], ci[b, 3], ci[b, 4]], [ci[b, 3], ci[b, 1], ci[b, 5]], [ci[b, 4], ci[b, 5], ci[b, 2]]])
            Iw = Iw - mass[b] * (np.dot(dc, dc) * np.eye(3) - np.outer(dc, dc))
            assert np.allclose(F, mass[b] * a_com, rtol=0, atol=1e-8 * big), (task, b, F - mass[b] * a_com)
            dL = Iw @ o["body_acc"][b, :3] + np.cross(w_b, Iw @ w_b)
            assert np.allclose(T, dL, rtol=0, atol=1e-8 * big), (task, b, T - dL)
        # (c) joint space: the projection of cfrc_int on each dof
        cdof = o["cdof"]
        lhs, contact_part = np.zeros(m.nv), np.zeros(m.nv)
        r2 = r.forward(q, v, _ctrl(spec, rng.uniform(-1, 1, m.nu)), qfrc=qfrc)      # no xfrc: cfrc_ext = contacts
        for j in range(m.nv):
            b = int(m.jnt_bodyid[j])
            f = r2["cfrc_int"][b]
            lhs[j] = cdof[j] @ np.concatenate([f[3:] + np.cross(xpos[b] - com, f[:3]), f[:3]])
            for c in subtree[b]:
                e = r2["cfrc_ext"][c]
                contact_part[j] += cdof[j] @ np.concatenate([e[3:] + np.cross(xpos[c] - com, e[:3]), e[:3]])
        rhs = r2["dof"][:, 0] + r2["passive"] + qfrc + r2["dof"][:, 1] - contact_part - \
            np.asarray(m.dof_armature, dtype=np.float64) * r2["dof"][:, 2]
        assert np.allclose(lhs, rhs, rtol=0, atol=1e-8 * max(1.0, np.abs(rhs).max())), (task, lhs - rhs)
    r.close()
    assert contacts >= 1, task


# ---------------------------------------------------------------------------------------------------------------------
# the serial fp32 core against the fp64 reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", list(CFG_TASKS))
def test_serial_core_matches_the_reference(emu, ref, bundled_only, cfg):
    """emu_forward_outputs (the kernels' source, serial) at the reference's states under random actions and applied
    forces, within forward_ref.REL of each output's magnitude (forward_ref.py states the error model); a sample outside it
    must be within 10x the reference's own jump under fp32-sized perturbations of the state, at most 2 of 10"""
    from loco_mujoco_b200 import modelpack
    env = make_task(CFG_TASKS[cfg])
    m, spec = env._model, env.task_spec()
    mb, tb = blobs(env)
    s = _emu(emu, modelpack.pack(m))
    r = fwr.ForwardSim(ref, mb, tb, env._model_user_features[0])
    p = fwr._p
    rng = np.random.RandomState(8)
    explained, constrained, worst = 0, 0, 0.0
    for q, v in _states(env, ref, 10, 3):
        q32, v32 = q.astype(np.float32).astype(np.float64), v.astype(np.float32).astype(np.float64)
        ctrl = _ctrl(spec, rng.uniform(-1, 1, m.nu))
        xfrc = rng.normal(0, 2, (m.nbody, 6)).astype(np.float32)
        qfrc = rng.normal(0, 2, m.nv).astype(np.float32)
        emu.emu_set_applied(s, p(xfrc), p(qfrc))
        got = fwr.emu_forward(emu, s, m.nv, m.nbody, q32, v32, ctrl)
        want = r.forward(q32, v32, ctrl, xfrc=xfrc.astype(np.float64), qfrc=qfrc.astype(np.float64))
        constrained += int(np.abs(want["cfrc_ext"]).max() > 1.0)
        ok = True
        for k in fwr.OUTPUTS:
            good, ratio = fwr.within(got[k], want[k], k)
            worst = max(worst, ratio)
            ok = ok and good
        if not ok:
            gap = r.sensitivity(q32, v32, ctrl, want)
            for k in fwr.OUTPUTS:
                assert fwr.within(got[k], want[k], k, gap[k])[0], (cfg, k)
            explained += 1
    emu.emu_set_applied(s, None, None)
    r.close()
    emu.emu_destroy(s)
    print("%s: worst error / bound %.3f, %d of 10 samples explained by the reference's jump" % (cfg, worst, explained))
    assert explained <= 2 and constrained >= 3, (cfg, explained, constrained)


def test_any_subset_of_outputs_gives_the_same_bits_and_non_finite_input_zero_rows(emu, bundled_only):
    from loco_mujoco_b200 import modelpack
    env = make_task("UnitreeA1.simple")
    m, spec = env._model, env.task_spec()
    s = _emu(emu, modelpack.pack(m))
    (q, v), = [(r[:m.nv].astype(np.float64), r[m.nv:2 * m.nv].astype(np.float64))
               for r in spec.table.reshape(-1, spec.table.shape[-1])[[37]]]
    ctrl = _ctrl(spec, np.linspace(-1, 1, m.nu))
    full = fwr.emu_forward(emu, s, m.nv, m.nbody, q, v, ctrl)
    assert all(np.all(np.isfinite(x)) for x in full.values())
    for k in fwr.OUTPUTS:
        one = fwr.emu_forward(emu, s, m.nv, m.nbody, q, v, ctrl, which=(k,))
        assert np.array_equal(one[k], full[k]), k
    for qq, vv, cc in ((np.where(np.arange(m.nv) == 3, np.nan, q), v, ctrl), (q, np.where(np.arange(m.nv) == 0, np.inf, v), ctrl),
                       (q, v, np.where(np.arange(m.nu) == 5, np.nan, ctrl))):
        out = fwr.emu_forward(emu, s, m.nv, m.nbody, qq, vv, cc)
        assert all(np.array_equal(x, np.zeros_like(x)) for x in out.values())
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


def test_forward_validates_its_arguments(monkeypatch):
    """dtype / shape / layout / device / overlap checks happen before the engine is called (no device needed)"""
    from loco_mujoco_b200 import engine as engine_mod
    calls = []
    eng = object.__new__(engine_mod.CudaEngine)
    eng.torch = types.SimpleNamespace(float32="float32", Tensor=_FakeTensor)
    eng.n_envs, eng.nq, eng.nbody, eng.action_dim, eng.device, eng.h, eng.launches = 4, 18, 14, 12, "cuda:0", None, 0
    eng.lib = types.SimpleNamespace(locosim_forward=lambda h, a, d, b, i, e, s: calls.append((a, d, b, i, e)) or 0)
    eng._stream = lambda: None
    monkeypatch.setattr(engine_mod, "_ptr", lambda t: None if t is None else id(t))
    base = 1 << 20
    act = _FakeTensor((4, 12), ptr=base)
    dof = _FakeTensor((4, 18, 3), ptr=base + 4096)
    acc = _FakeTensor((4, 14, 6), ptr=base + 8192)
    cint = _FakeTensor((4, 14, 6), ptr=base + 16384)
    cext = _FakeTensor((4, 14, 6), ptr=base + 24576)
    assert eng.forward(act) == {} and calls == []                 # nothing asked for: nothing launched
    got = eng.forward(act, dof=dof, body_acc=acc, cfrc_int=cint, cfrc_ext=cext)
    assert got == dict(dof=dof, body_acc=acc, cfrc_int=cint, cfrc_ext=cext)
    assert calls == [(id(act), id(dof), id(acc), id(cint), id(cext))]
    assert eng.forward(act, cfrc_ext=cext) == dict(cfrc_ext=cext) and calls[-1] == (id(act), None, None, None, id(cext))
    for bad in (_FakeTensor((4, 11)), _FakeTensor((3, 12)), _FakeTensor((4, 12), "float64"), _FakeTensor((4, 12), contiguous=False),
                _FakeTensor((4, 12), device="cuda:1"), np.zeros((4, 12), np.float32), None):
        with pytest.raises(ValueError):
            eng.forward(bad, dof=dof)
    for kw in (dict(dof=_FakeTensor((4, 18, 2))), dict(body_acc=_FakeTensor((4, 13, 6))), dict(cfrc_int=_FakeTensor((4, 14, 3))),
               dict(cfrc_ext=_FakeTensor((4, 14, 6), "float64"))):
        with pytest.raises(ValueError):
            eng.forward(act, **kw)
    # overlapping buffers are refused: two outputs, and an output with the action
    with pytest.raises(ValueError):
        eng.forward(act, body_acc=acc, cfrc_int=_FakeTensor((4, 14, 6), ptr=base + 8192 + 4 * 4 * 14 * 6 - 4))
    with pytest.raises(ValueError):
        eng.forward(act, dof=_FakeTensor((4, 18, 3), ptr=base + 4 * 4 * 12 - 4))
    assert len(calls) == 2


def test_4ages_all_refuses_forward_dynamics(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    env = LocoEnv.make("HumanoidTorque4Ages.walk.all.real", num_envs=8, debug=True)
    with pytest.raises(NotImplementedError):
        env.forward_dynamics(None)
