"""Body outputs (MuJoCo's xpos / xquat / mj_objectVelocity, include/locosim.h locosim_set_body_outputs) without a GPU: the
fp64 reference (tests/body_outputs_ref.py) against a hand-computed model, the serial build of the CUDA core against that
reference, and the host-side rules."""
import types

import numpy as np
import pytest

import body_outputs_ref
from body_outputs_ref import BodyRef, compare
from full_body import make_variant
from helpers import make_env, oracle_env

TASKS = ["UnitreeA1.simple", "HumanoidTorque.run", "Talos.walk", "Atlas.walk+arms+back", "Talos.walk+arms"]

# fp32 tolerance of compare() (errors relative to the magnitudes that set the rounding). fp32's unit round-off is 6e-8; a
# body pose is a chain of up to ~10 quaternion products and vector rotations from the root, a velocity a sum over up to 31
# dofs of cdof * qvel plus the shift from the CoM to the body origin: a few hundred round-offs at most, i.e. ~1e-5 of the
# magnitudes. The central differences of the reference add O(eps^2) + O(1e-16 / eps) = 1e-10.
TOL = 2e-5


def _hinge_model(tmp_path):
    from loco_mujoco_b200 import mjcf
    xml = tmp_path / "m.xml"
    xml.write_text("""<mujoco><worldbody>
      <body name="base" pos="0 0 1"><joint name="root_z" type="slide" axis="0 0 1"/>
        <geom type="sphere" size="0.1" mass="1"/>
        <body name="link" pos="0.5 0 0"><joint name="hinge" type="hinge" axis="0 1 0" pos="-0.3 0 0"/>
          <geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.03" mass="0.3"/></body>
      </body></worldbody></mujoco>""")
    return mjcf.compile_model(mjcf.XmlHandle(str(xml)))


def _hand(z, th, zd, thd):
    """the hinge model by hand: the link's origin circles the anchor (0.2, 0, 1 + z) at radius 0.3 about world y"""
    s, c = np.sin(th), np.cos(th)
    base = [0, 0, 1 + z, 1, 0, 0, 0, 0, 0, 0, 0, 0, zd]
    link = [0.2 + 0.3 * c, 0, 1 + z - 0.3 * s, np.cos(th / 2), 0, np.sin(th / 2), 0, 0, thd, 0,
            -0.3 * s * thd, 0, zd - 0.3 * c * thd]
    return np.array([[0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0], base, link])


def test_reference_matches_a_hand_computed_hinge(oracle, tmp_path):
    m = _hinge_model(tmp_path)
    assert m.body_names == ["world", "base", "link"]
    ref = BodyRef(oracle, m)
    for z, th, zd, thd in [(0.0, 0.0, 0.0, 1.0), (0.3, 0.7, -1.5, 2.5), (-0.2, -2.4, 0.4, -7.0)]:
        got, want = ref([z, th], [zd, thd]), _hand(z, th, zd, thd)
        assert np.abs(got - want).max() < 1e-8, np.abs(got - want).max()
    ref.close()


def test_serial_core_on_the_hinge(emu, oracle, tmp_path):
    from loco_mujoco_b200 import modelpack
    body_outputs_ref.emu_bind(emu)
    m = _hinge_model(tmp_path)
    ints, reals = modelpack.pack(m)
    p = body_outputs_ref._p
    ints, reals = np.ascontiguousarray(ints, dtype=np.int32), np.ascontiguousarray(reals, dtype=np.float64)
    sim = emu.emu_create(p(ints), len(ints), p(reals), len(reals))
    assert sim
    q, v = np.array([0.3, 0.7]), np.array([-1.5, 2.5])
    emu.emu_reset(sim, p(q), p(v))
    got = body_outputs_ref.emu_body(emu, sim, m.nbody)
    emu.emu_destroy(sim)
    want = _hand(*q, *v)
    assert np.array_equal(got[0], want[0])          # the world row is exact
    assert max(compare(got, want)) < TOL


def _states(oracle, env, rng, n_table=6, n_roll=8):
    """(qpos, qvel) pairs: rows of the reset table, and the states of an oracle rollout under U(-1, 1) actions (until it falls)"""
    spec = env.task_spec()
    nv = env._model.nv
    table = spec.table.reshape(-1, spec.table.shape[-1])
    out = [(table[i, :nv], table[i, nv:2 * nv]) for i in rng.randint(len(table), size=n_table)]
    oe = oracle_env(oracle, env)
    oe.reset_to(rng.randint(env.trajectories.number_of_trajectories), rng.randint(env.trajectories.trajectory_length - 1))
    for _ in range(n_roll):
        _, _, done = oe.step(rng.uniform(-1, 1, env._model.nu))
        out.append(oe.get_state())
        if done:
            break
    oe.close()
    return out


@pytest.mark.parametrize("task", TASKS)
def test_serial_core_matches_the_reference(emu, oracle, bundled_only, task):
    """The serial build of the CUDA core (same source as the kernels) against the fp64 reference at reset-table states and
    at states of oracle rollouts under random actions (velocities there reach tens of rad/s)."""
    from loco_mujoco_b200 import modelpack
    body_outputs_ref.emu_bind(emu)
    env = make_variant(task)
    m = env._model
    ints, reals = modelpack.pack(m)
    p = body_outputs_ref._p
    ints, reals = np.ascontiguousarray(ints, dtype=np.int32), np.ascontiguousarray(reals, dtype=np.float64)
    sim = emu.emu_create(p(ints), len(ints), p(reals), len(reals))
    assert sim
    ref = BodyRef(oracle, m)
    rng = np.random.RandomState(7)
    worst = np.zeros(4)
    for q, v in _states(oracle, env, rng):
        q, v = np.ascontiguousarray(q, dtype=np.float64), np.ascontiguousarray(v, dtype=np.float64)
        emu.emu_reset(sim, p(q), p(v))
        got = body_outputs_ref.emu_body(emu, sim, m.nbody)
        want = ref(q, v)
        assert np.array_equal(got[0], want[0])
        worst = np.maximum(worst, compare(got, want))
    emu.emu_destroy(sim)
    ref.close()
    assert worst.max() < TOL, (task, worst)


# ---------------------------------------------------------------------------------------------------------------------
# host logic
# ---------------------------------------------------------------------------------------------------------------------
class _FakeTensor:
    def __init__(self, shape, dtype="float32", contiguous=True, device="cuda:0"):
        self.shape, self.dtype, self._c, self.device = shape, dtype, contiguous, device

    def is_contiguous(self):
        return self._c


def test_set_body_outputs_validates_its_arguments(monkeypatch):
    """dtype / shape / layout / device checks happen before the engine is called (no device needed)"""
    from loco_mujoco_b200 import engine as engine_mod
    calls = []
    eng = object.__new__(engine_mod.CudaEngine)
    eng.torch = types.SimpleNamespace(float32="float32")
    eng.n_envs, eng.nbody, eng.device, eng.h = 4, 3, "cuda:0", None
    eng.lib = types.SimpleNamespace(locosim_set_body_outputs=lambda h, b, n: calls.append((b, n)) or 0,
                                    locosim_kernels_per_step=lambda h: 1)
    monkeypatch.setattr(engine_mod, "_ptr", lambda t: None if t is None else id(t))
    ok_b, ok_n = _FakeTensor((4, 3, 13)), _FakeTensor((4, 3, 13))
    eng.set_body_outputs(ok_b, ok_n)
    eng.set_body_outputs(None, ok_n)
    eng.set_body_outputs(ok_b)
    eng.set_body_outputs()
    assert calls == [(id(ok_b), id(ok_n)), (None, id(ok_n)), (id(ok_b), None), (None, None)]
    assert eng._body_out == (None, None)
    for bad in (_FakeTensor((4, 3, 12)), _FakeTensor((4, 4, 13)), _FakeTensor((3, 3, 13)), _FakeTensor((4, 3, 13), "float64"),
                _FakeTensor((4, 3, 13), contiguous=False), _FakeTensor((4, 3, 13), device="cuda:1")):
        with pytest.raises(ValueError):
            eng.set_body_outputs(bad, None)
        with pytest.raises(ValueError):
            eng.set_body_outputs(ok_b, bad)
    assert len(calls) == 4
    assert engine_mod.BODY_DIM == 13


class _RecordingEngine:
    """Stands in for CudaEngine on a CPU-only box: records what the env registers."""
    made = []

    def __init__(self, model_blobs, task_blobs, n_envs, device=0, **kw):
        import torch
        self.device, self.n_envs, self.calls = torch.device("cpu"), n_envs, []
        _RecordingEngine.made.append(self)

    def set_body_outputs(self, body=None, next_body=None):
        self.calls.append((body, next_body))

    def set_param_pool(self, pool):
        pass

    def close(self):
        pass


def test_body_state_is_lazy_and_survives_an_engine_rebuild(bundled_only, monkeypatch):
    from loco_mujoco_b200 import engine as engine_mod
    monkeypatch.setattr(engine_mod, "CudaEngine", _RecordingEngine)
    _RecordingEngine.made = []
    env = make_env("UnitreeA1.simple", num_envs=5)
    eng = env._get_engine()
    assert eng.calls == []                                       # nothing registered until a tensor is asked for
    nb = env._model.nbody
    b = env.body_state
    n = env.next_body_state
    assert tuple(b.shape) == tuple(n.shape) == (5, nb, 13) and b.dtype == n.dtype and str(b.dtype) == "torch.float32"
    assert b.is_contiguous() and n.is_contiguous() and b.data_ptr() != n.data_ptr()
    assert len(eng.calls) == 1 and eng.calls[0][0] is b and eng.calls[0][1] is n     # both at once, on first access
    assert env.body_state is b and env.next_body_state is n and len(eng.calls) == 1
    # layout: row body_index(name) of env i is b[i, body_index(name)]
    assert env.body_index("trunk") == env._model.body_names.index("trunk")
    env.set_launch_geometry(4)                                   # rebuilds the engine: the same tensors are registered again
    eng2 = env._get_engine()
    assert eng2 is not eng and len(eng2.calls) == 1 and eng2.calls[0][0] is b and eng2.calls[0][1] is n


def test_next_body_state_alone_registers_both(bundled_only, monkeypatch):
    from loco_mujoco_b200 import engine as engine_mod
    monkeypatch.setattr(engine_mod, "CudaEngine", _RecordingEngine)
    env = make_env("HumanoidTorque.run", num_envs=3)
    n = env.next_body_state
    eng = env._get_engine()
    assert len(eng.calls) == 1 and eng.calls[0][1] is n and eng.calls[0][0] is env.body_state


def test_4ages_all_refuses_body_outputs(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    env = LocoEnv.make("HumanoidTorque4Ages.walk.all.real", num_envs=8, debug=True)
    for get in (lambda: env.body_state, lambda: env.next_body_state):
        with pytest.raises(NotImplementedError):
            get()
