"""Saved simulation states without a GPU (include/locosim.h locosim_save_state / locosim_load_state; CudaEngine.save_state /
load_state / state_layout; LocoEnv.save_state / load_state): the argument checks, the row layout against the header's
LS_STATE_* macros (compiled), the refusals, and the restated counter-based draws the GPU tier predicts forks with."""
import os
import subprocess
import types

import numpy as np
import pytest

import sim_state_ref as ref
from helpers import GOLDEN_TASKS, ROOT, make_env


class _FakeTensor:
    _next = [1]

    def __init__(self, shape, dtype="float32", contiguous=True, device="cuda:0"):
        self.shape, self.dtype, self._c, self.device = tuple(shape), dtype, contiguous, device
        self._ptr = _FakeTensor._next[0] << 32          # (far apart: no two fake buffers overlap)
        _FakeTensor._next[0] += 1

    def is_contiguous(self):
        return self._c

    def data_ptr(self):
        return self._ptr


N, NQ, D = 4, 18, 37


@pytest.fixture
def eng(monkeypatch):
    from loco_mujoco_b200 import engine as engine_mod
    eng = object.__new__(engine_mod.CudaEngine)
    eng.torch = types.SimpleNamespace(float32="float32", int32="int32",
                                      empty=lambda shape, dtype, device: _FakeTensor(shape, dtype, device=device))
    eng.n_envs, eng.nq, eng.obs_dim, eng.device, eng.h = N, NQ, D, "cuda:0", None
    eng.state_words = engine_mod.state_layout(NQ, D)["words"][1]
    eng._body_out, eng._ref_out, eng.launches = (None, None), (None, None), 0
    eng.calls = []
    eng.lib = types.SimpleNamespace(
        locosim_save_state=lambda h, o, s, st: eng.calls.append(("save", o, s)) or 0,
        locosim_load_state=lambda h, s, m, r, o, st: eng.calls.append(("load", s, m, r, o)) or 0)
    eng._stream = lambda: None
    monkeypatch.setattr(engine_mod, "_ptr", lambda t: None if t is None else t.data_ptr())
    return eng


def _bad(shape, dtype):
    other = "float64" if dtype == "float32" else "int64"
    return [_FakeTensor(shape[:-1] + (shape[-1] - 1,), dtype), _FakeTensor(shape[1:], dtype), _FakeTensor(shape, other),
            _FakeTensor(shape, "float32" if dtype == "int32" else "int32"), _FakeTensor(shape, dtype, contiguous=False),
            _FakeTensor(shape, dtype, device="cuda:1"), _FakeTensor(shape, dtype, device="cpu"),
            np.zeros(shape, np.float32 if dtype == "float32" else np.int32)]


def test_save_state_validates_its_arguments(eng):
    W = eng.state_words
    obs, out = _FakeTensor((N, D)), _FakeTensor((N, W), "int32")
    assert eng.save_state(obs, out) is out
    fresh = eng.save_state(obs)
    assert fresh.shape == (N, W) and fresh.dtype == "int32"
    assert eng.calls == [("save", obs.data_ptr(), out.data_ptr()), ("save", obs.data_ptr(), fresh.data_ptr())]
    for bad in _bad((N, D), "float32") + [None, _FakeTensor((N + 1, D))]:
        with pytest.raises(ValueError, match="obs"):
            eng.save_state(bad, out)
    for bad in _bad((N, W), "int32") + [_FakeTensor((N + 1, W), "int32")]:
        with pytest.raises(ValueError, match="out"):
            eng.save_state(obs, bad)
    # the observation and the rows must not share bytes
    alias = _FakeTensor((N, W), "int32")
    alias._ptr = obs.data_ptr() + 4
    with pytest.raises(ValueError, match="overlap"):
        eng.save_state(obs, alias)
    assert len(eng.calls) == 2


def test_load_state_validates_its_arguments(eng):
    W = eng.state_words
    rows, idx, obs = _FakeTensor((N, W), "int32"), _FakeTensor((N,), "int32"), _FakeTensor((N, D))
    eng.load_state(rows)
    eng.load_state(rows, idx, obs)
    bank = _FakeTensor((3 * N, W), "int32")
    eng.load_state(bank, idx)
    small = _FakeTensor((1, W), "int32")
    eng.load_state(small, idx)
    assert eng.calls == [("load", rows.data_ptr(), N, None, None), ("load", rows.data_ptr(), N, idx.data_ptr(), obs.data_ptr()),
                         ("load", bank.data_ptr(), 3 * N, idx.data_ptr(), None), ("load", small.data_ptr(), 1, idx.data_ptr(), None)]
    for bad in _bad((N, W), "int32") + [None, _FakeTensor((0, W), "int32"), _FakeTensor((N, W, 1), "int32")]:
        with pytest.raises(ValueError, match="rows"):
            eng.load_state(bad, idx)
    # without an index, one row per env
    with pytest.raises(ValueError, match="one row per env"):
        eng.load_state(bank)
    for bad in _bad((N,), "int32") + [_FakeTensor((N + 1,), "int32"), _FakeTensor((N, 1), "int32")]:
        with pytest.raises(ValueError, match="index"):
            eng.load_state(rows, bad)
    for bad in _bad((N, D), "float32"):
        with pytest.raises(ValueError, match="obs_out"):
            eng.load_state(rows, idx, bad)
    alias = _FakeTensor((N, D))
    alias._ptr = rows.data_ptr() + 16
    with pytest.raises(ValueError, match="overlap"):
        eng.load_state(rows, idx, alias)
    assert len(eng.calls) == 4


def _header_layout(tmp_path, cases):
    """{(nv, obs_dim): {field: offset}} and W from the header's macros, compiled and run on the host"""
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stdlib.h>\n#include "locosim.h"\n'
                   "int main(int c, char** v) { int nv = atoi(v[1]), d = atoi(v[2]);\n"
                   '  printf("%d %d %d %d %d %d %d %d %d %d %d %d %d %d\\n", LS_STATE_TAG, LS_STATE_EPISODE, LS_STATE_DR_ROW,'
                   " LS_STATE_CURSOR, LS_STATE_ANGLE, LS_STATE_EP, LS_STATE_GOAL, LS_STATE_QPOS(nv), LS_STATE_QVEL(nv),"
                   " LS_STATE_WARMSTART(nv), LS_STATE_OBS(nv), LS_STATE_WORDS(nv, d), LS_STATE_VERSION, 0);\n"
                   "  return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = {}
    for nv, d in cases:
        vals = [int(x) for x in subprocess.check_output([str(exe), str(nv), str(d)]).split()]
        out[(nv, d)] = vals
    return out


def _bundled_dims():
    from full_body import VARIANTS, make_variant
    from position_mode import make_position
    dims = {}
    for task in GOLDEN_TASKS:
        env = make_env(task, num_envs=2)
        dims[task] = (env._model.nq, env.task_spec().obs_dim)
    for name in VARIANTS:
        env = make_variant(name, num_envs=2)
        dims[name] = (env._model.nq, env.task_spec().obs_dim)
    for task in ("UnitreeA1.simple", "UnitreeA1.hard"):
        env = make_position(task, num_envs=2)
        dims[task + "+position"] = (env._model.nq, env.task_spec().obs_dim)
    return dims


def test_state_layout_matches_the_header(bundled_only, tmp_path):
    """engine.state_layout agrees with LS_STATE_* for every bundled model and the full-body and position fixtures; the row
    is a whole number of 16-byte words and its fields tile it without overlap."""
    from loco_mujoco_b200.engine import state_layout
    dims = _bundled_dims()
    hdr = _header_layout(tmp_path, sorted(set(dims.values())))
    for name, (nq, d) in dims.items():
        lay = state_layout(nq, d)
        tag, episode, dr_row, cursor, angle, ep, goal, qpos, qvel, ws, obs, words, version, _ = hdr[(nq, d)]
        assert version == 0x4C530001
        assert {k: v[0] for k, v in lay.items() if k != "words"} == dict(
            tag=tag, episode=episode, dr_row=dr_row, cursor=cursor, angle=angle, ep=ep, goal=goal, qpos=qpos, qvel=qvel,
            qacc_warmstart=ws, obs=obs), name
        W = lay["words"][1]
        assert W == words and W % 4 == 0, name
        used = np.zeros(W, int)
        for k, (off, n) in lay.items():
            if k != "words":
                used[off:off + n] += 1
        assert used.max() == 1 and used[obs + d:].sum() == 0 and W - (obs + d) < 4, name


def test_4ages_all_refuses_saved_states(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    env = LocoEnv.make("HumanoidTorque4Ages.walk.all.real", num_envs=8, debug=True)
    with pytest.raises(NotImplementedError, match="save_state"):
        env.save_state()
    with pytest.raises(NotImplementedError, match="load_state"):
        env.load_state(None)


@pytest.mark.parametrize("num_envs", [None, 4])
def test_saved_states_need_a_reset_first(bundled_only, num_envs):
    """Before the first reset() there is no observation to save (or to keep for envs a load leaves untouched); refused
    before any engine is created."""
    env = make_env("UnitreeA1.simple", num_envs=num_envs)
    with pytest.raises(RuntimeError, match="reset"):
        env.save_state()
    with pytest.raises(RuntimeError, match="reset"):
        env.load_state(None)
    assert env._engine is None


def test_restated_draws():
    """The restated draws: deterministic, in range, and different for neighbouring envs and episodes (pinned values guard
    the 64-bit arithmetic against a silent change)."""
    seed = 3
    a = [ref.draw_reset(seed, g, e, 7, 500) for g in range(64) for e in range(4)]
    assert all(0 <= t < 7 and 0 <= s < 500 for t, s in a)
    assert len(set(a)) > 200
    ang = np.array([ref.draw_rot_angle(seed, g, e) for g in range(64) for e in range(4)])
    assert ang.dtype == np.float32 and ang.min() >= 0 and ang.max() < 2 * np.pi
    rows = [ref.draw_pool_row(seed, g, e, 5) for g in range(64) for e in range(4)]
    assert set(rows) == set(range(5)) and ref.draw_pool_row(seed, 1, 2, 1) == 0
    assert ref.mix64(0) == 0xE220A8397B1DCDAF
