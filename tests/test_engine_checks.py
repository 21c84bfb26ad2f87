"""CudaEngine's argument checks without a GPU: set_state and set_goal copy every env's whole rows from the pointers they are
given (include/locosim.h locosim_set_state: n_envs * nq floats each, locosim_set_goal: n_envs * 4), so a tensor of the
wrong shape or on another device is refused before the engine is called."""
import types

import numpy as np
import pytest


class _FakeTensor:
    def __init__(self, shape, dtype="float32", contiguous=True, device="cuda:0"):
        self.shape, self.dtype, self._c, self.device = shape, dtype, contiguous, device

    def is_contiguous(self):
        return self._c


@pytest.fixture
def eng(monkeypatch):
    from loco_mujoco_b200 import engine as engine_mod
    eng = object.__new__(engine_mod.CudaEngine)
    eng.torch = types.SimpleNamespace(float32="float32", Tensor=_FakeTensor)
    eng.n_envs, eng.nq, eng.device, eng.h = 4, 18, "cuda:0", None
    eng.calls = []
    eng.lib = types.SimpleNamespace(locosim_set_state=lambda h, q, v, w, s: eng.calls.append(("state", q, v, w)) or 0,
                                    locosim_set_goal=lambda h, g, s: eng.calls.append(("goal", g)) or 0)
    eng._stream = lambda: None
    monkeypatch.setattr(engine_mod, "_ptr", lambda t: None if t is None else id(t))
    return eng


def _bad(shape):
    return [_FakeTensor(shape[:-1] + (shape[-1] - 1,)), _FakeTensor((shape[0] - 1,) + shape[1:]), _FakeTensor(shape[1:]),
            _FakeTensor(shape, "float64"), _FakeTensor(shape, contiguous=False), _FakeTensor(shape, device="cuda:1"),
            _FakeTensor(shape, device="cpu"), np.zeros(shape, np.float32)]


def test_set_state_validates_its_arguments(eng):
    q, v, w = (_FakeTensor((4, 18)) for _ in range(3))
    eng.set_state(q, v, w)
    eng.set_state(q, v)
    eng.set_state(None, v)
    assert eng.calls == [("state", id(q), id(v), id(w)), ("state", id(q), id(v), None), ("state", None, id(v), None)]
    for bad in _bad((4, 18)):
        for args in ((bad, v), (q, bad), (q, v, bad)):
            with pytest.raises(ValueError):
                eng.set_state(*args)
    assert len(eng.calls) == 3


def test_set_goal_validates_its_argument(eng):
    g = _FakeTensor((4, 4))
    eng.set_goal(g)
    assert eng.calls == [("goal", id(g))]
    for bad in _bad((4, 4)) + [None]:
        with pytest.raises(ValueError, match="goal"):
            eng.set_goal(bad)
    assert len(eng.calls) == 1
