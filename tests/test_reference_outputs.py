"""Reference outputs (the mocap clip's body outputs, include/locosim.h locosim_set_reference_outputs /
locosim_create_dataset_bodies; LocoEnv.reference_body_state / next_reference_body_state / create_dataset_bodies) without a
GPU: the serial build of the CUDA core against the fp64 reference at the fp64 reset state (tests/reference_outputs_ref.py),
the dataset's row mapping, and the host-side rules."""
import types

import numpy as np
import pytest

import body_outputs_ref
import reference_outputs_ref
from body_outputs_ref import BodyRef, compare
from full_body import make_variant, obs_from_state
from helpers import make_env

TOL = 2e-5          # as tests/test_body_outputs.py: the same core (body_outputs) on a state of the same magnitudes

# (variant name, make_env keywords, rotation angles): UnitreeA1 under setup_random_rot with angles away from 0 and around the
# yaw's wrap; the humanoids have no such option (the angle is ignored)
CASES = [("UnitreeA1.simple", dict(setup_random_rot=True), [0.0, 1.3, 3.1, 4.0, 6.2]),
         ("HumanoidTorque.run", {}, [0.0, 2.0]),
         ("Talos.walk", {}, [0.0]),
         ("Atlas.walk+arms", {}, [0.0])]


def _emu_sim(emu, model):
    from loco_mujoco_b200 import modelpack
    ints, reals = modelpack.pack(model)
    ints, reals = np.ascontiguousarray(ints, dtype=np.int32), np.ascontiguousarray(reals, dtype=np.float64)
    sim = emu.emu_create(body_outputs_ref._p(ints), len(ints), body_outputs_ref._p(reals), len(reals))
    assert sim
    return sim, (ints, reals)


@pytest.mark.parametrize("task,kw,angles", CASES, ids=[c[0] for c in CASES])
def test_serial_core_matches_the_reference_at_the_reset_state(emu, oracle, bundled_only, task, kw, angles):
    """Table rows of every trajectory, first and last samples included, under each angle: the serial core's reference row
    against BodyRef at the fp64 reset state of the same (fp32) table row."""
    reference_outputs_ref.emu_bind(emu)
    env = make_variant(task, **kw)
    m, spec = env._model, env.task_spec()
    assert (spec.random_rot[0] >= 0) == bool(kw.get("setup_random_rot"))
    sim, keep = _emu_sim(emu, m)
    ref = BodyRef(oracle, m)
    n_traj, T = spec.table.shape[:2]
    rng = np.random.RandomState(11)
    picks = [(0, 0), (n_traj - 1, T - 1)] + [(rng.randint(n_traj), rng.randint(T)) for _ in range(4)]
    worst = np.zeros(4)
    for angle in angles:
        for tj, sp in picks:
            row = spec.table[tj, sp].astype(np.float32)
            got = reference_outputs_ref.emu_reference_row(emu, sim, spec, row, m.nbody, angle)
            q, v = reference_outputs_ref.reset_state(spec, row, m.nv, np.float64(np.float32(angle)))
            want = ref(q, v)
            assert np.array_equal(got[0], want[0])
            assert np.abs(got[1, 0:2]).max() < 1e-6            # the root body stands at x = y = 0
            worst = np.maximum(worst, compare(got, want))
    emu.emu_destroy(sim)
    ref.close()
    assert worst.max() < TOL, (task, worst)


@pytest.mark.parametrize("task", ["HumanoidTorque.run", "Talos.walk"])
def test_dataset_rows_against_the_reference(emu, oracle, bundled_only, task):
    """Dataset row r of locosim_create_dataset is (traj, sample) = divmod(r, traj_len - 1) -> (traj, sample + 1): checked
    against the host create_dataset(); the reference rows of both samples (angle 0, the model's own parameters) against
    BodyRef, on a sample of rows that includes every trajectory's last transition."""
    reference_outputs_ref.emu_bind(emu)
    env = make_env(task)
    m, spec = env._model, env.task_spec()
    nv = m.nv
    host = env.create_dataset()
    n_traj, T = spec.table.shape[:2]
    per = T - 1
    assert len(host["states"]) == n_traj * per
    rng = np.random.RandomState(3)
    rows = sorted(set([tj * per + per - 1 for tj in range(n_traj)] + [0] + list(rng.randint(n_traj * per, size=4))))
    sim, keep = _emu_sim(emu, m)
    ref = BodyRef(oracle, m)
    worst = np.zeros(4)
    for r in rows:
        tj, sp = divmod(r, per)
        for col, k in (("states", sp), ("next_states", sp + 1)):
            tr = spec.table[tj, k]
            assert np.abs(host[col][r] - obs_from_state(spec, tr[:nv], tr[nv:2 * nv])).max() < 1e-5
            got = reference_outputs_ref.emu_reference_row(emu, sim, spec, tr, m.nbody, 0.0)
            want = ref(*reference_outputs_ref.reset_state(spec, tr.astype(np.float32), nv, 0.0))
            worst = np.maximum(worst, compare(got, want))
        assert bool(host["last"][r]) == (sp == per - 1)
    emu.emu_destroy(sim)
    ref.close()
    assert worst.max() < TOL, worst


# ---------------------------------------------------------------------------------------------------------------------
# host logic
# ---------------------------------------------------------------------------------------------------------------------
class _FakeTensor:
    def __init__(self, shape, dtype="float32", contiguous=True, device="cuda:0"):
        self.shape, self.dtype, self._c, self.device = shape, dtype, contiguous, device

    def is_contiguous(self):
        return self._c


def test_set_reference_outputs_validates_its_arguments(monkeypatch):
    """dtype / shape / layout / device checks happen before the engine is called (no device needed)"""
    from loco_mujoco_b200 import engine as engine_mod
    calls = []
    eng = object.__new__(engine_mod.CudaEngine)
    eng.torch = types.SimpleNamespace(float32="float32")
    eng.n_envs, eng.nbody, eng.device, eng.h = 4, 3, "cuda:0", None
    eng.lib = types.SimpleNamespace(locosim_set_reference_outputs=lambda h, r, n: calls.append((r, n)) or 0,
                                    locosim_kernels_per_step=lambda h: 1)
    monkeypatch.setattr(engine_mod, "_ptr", lambda t: None if t is None else id(t))
    ok_r, ok_n = _FakeTensor((4, 3, 13)), _FakeTensor((4, 3, 13))
    eng.set_reference_outputs(ok_r, ok_n)
    eng.set_reference_outputs(None, ok_n)
    eng.set_reference_outputs(ok_r)
    eng.set_reference_outputs()
    assert calls == [(id(ok_r), id(ok_n)), (None, id(ok_n)), (id(ok_r), None), (None, None)]
    assert eng._ref_out == (None, None)
    for bad in (_FakeTensor((4, 3, 12)), _FakeTensor((4, 4, 13)), _FakeTensor((3, 3, 13)), _FakeTensor((4, 3, 13), "float64"),
                _FakeTensor((4, 3, 13), contiguous=False), _FakeTensor((4, 3, 13), device="cuda:1")):
        with pytest.raises(ValueError):
            eng.set_reference_outputs(bad, None)
        with pytest.raises(ValueError):
            eng.set_reference_outputs(ok_r, bad)
    assert len(calls) == 4
    assert "locosim_set_reference_outputs" in engine_mod.EXPORTED_SYMBOLS
    assert "locosim_create_dataset_bodies" in engine_mod.EXPORTED_SYMBOLS


class _RecordingEngine:
    """Stands in for CudaEngine on a CPU-only box: records what the env registers."""
    made = []

    def __init__(self, model_blobs, task_blobs, n_envs, device=0, **kw):
        import torch
        self.device, self.n_envs, self.calls = torch.device("cpu"), n_envs, []
        _RecordingEngine.made.append(self)

    def set_reference_outputs(self, ref=None, next_ref=None):
        self.calls.append((ref, next_ref))

    def set_time_limit(self, *args):
        pass

    def set_param_pool(self, pool):
        pass

    def close(self):
        pass


def test_reference_needs_a_moving_cursor(bundled_only, monkeypatch):
    """Without reward_type="tracking" or truncate_at_trajectory_end=True the cursor never leaves the reset sample: the
    facade refuses on first access, and the message names both ways out."""
    from loco_mujoco_b200 import engine as engine_mod
    monkeypatch.setattr(engine_mod, "CudaEngine", _RecordingEngine)
    env = make_env("UnitreeA1.simple", num_envs=4)
    for get in (lambda: env.reference_body_state, lambda: env.next_reference_body_state):
        with pytest.raises(ValueError) as err:
            get()
        assert "tracking" in str(err.value) and "truncate_at_trajectory_end" in str(err.value)
    assert env._reference_body_state is None
    # either option is enough
    for kw in (dict(reward_type="tracking"), dict(truncate_at_trajectory_end=True)):
        e = make_env("UnitreeA1.simple", num_envs=4, **kw)
        assert tuple(e.reference_body_state.shape) == (4, e._model.nbody, 13)


def test_reference_state_is_lazy_and_survives_an_engine_rebuild(bundled_only, monkeypatch):
    from loco_mujoco_b200 import engine as engine_mod
    monkeypatch.setattr(engine_mod, "CudaEngine", _RecordingEngine)
    env = make_env("UnitreeA1.simple", num_envs=5, truncate_at_trajectory_end=True)
    eng = env._get_engine()
    assert eng.calls == []                                       # nothing registered until a tensor is asked for
    nb = env._model.nbody
    n = env.next_reference_body_state
    r = env.reference_body_state
    assert tuple(r.shape) == tuple(n.shape) == (5, nb, 13) and str(r.dtype) == str(n.dtype) == "torch.float32"
    assert r.is_contiguous() and n.is_contiguous() and r.data_ptr() != n.data_ptr()
    assert len(eng.calls) == 1 and eng.calls[0][0] is r and eng.calls[0][1] is n     # both at once, on first access
    # rows are the model's body indices, as in body_state
    assert env.body_index("trunk") == env._model.body_names.index("trunk") < nb
    env.set_launch_geometry(4)                                   # rebuilds the engine: the same tensors are registered again
    eng2 = env._get_engine()
    assert eng2 is not eng and len(eng2.calls) == 1 and eng2.calls[0][0] is r and eng2.calls[0][1] is n


def test_create_dataset_bodies_returns_both_halves(bundled_only, monkeypatch):
    from loco_mujoco_b200 import engine as engine_mod
    monkeypatch.setattr(engine_mod, "CudaEngine", _RecordingEngine)
    env = make_env("HumanoidTorque.run", num_envs=3)
    eng = env._get_engine()
    eng.create_dataset_bodies = lambda: ("b", "n")
    assert env.create_dataset_bodies() == dict(body_states="b", next_body_states="n")


def test_4ages_all_refuses_reference_outputs(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    env = LocoEnv.make("HumanoidTorque4Ages.walk.all.real", num_envs=8, debug=True, truncate_at_trajectory_end=True)
    for get in (lambda: env.reference_body_state, lambda: env.next_reference_body_state, env.create_dataset_bodies):
        with pytest.raises(NotImplementedError):
            get()
