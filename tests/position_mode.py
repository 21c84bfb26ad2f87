"""UnitreeA1 under PD position control (action_mode "position" / "position_difference"), and what its tests share. Test
infrastructure only.

The compiled position models are data fixtures under tests/golden/position (tools/build_assets.py
UnitreeA1.simple+position UnitreeA1.hard+position); importing this module adds that directory to
LOCO_MUJOCO_B200_ASSET_PATH. No reference golden covers position mode (the reference's own tests run torque mode): its tests
compare the engine with the fp64 oracle, whose actuation evaluates the same gain / bias / clamp formula for every actuator."""
import os

from helpers import GOLDEN, make_env

FIXTURES = os.path.join(GOLDEN, "position")
if FIXTURES not in os.environ.get("LOCO_MUJOCO_B200_ASSET_PATH", "").split(os.pathsep):
    os.environ["LOCO_MUJOCO_B200_ASSET_PATH"] = os.pathsep.join(
        [p for p in (os.environ.get("LOCO_MUJOCO_B200_ASSET_PATH"), FIXTURES) if p])

# the position actuators of unitree_a1_position.xml: kp and forcerange from default class a1, ctrlrange per joint class
KP, FORCE = 100.0, 33.5
CTRLRANGE = {"hip": (-0.802851, 0.802851), "thigh": (-1.0472, 4.18879), "calf": (-2.69653, -0.916298)}


def make_position(task="UnitreeA1.simple", mode="position", **kw):
    """make_env of UnitreeA1 in a position action mode"""
    return make_env(task, action_mode=mode, **kw)


def compile_xml(xml):
    """(compiled model, ModelPack blobs) of an MJCF string"""
    import tempfile
    from loco_mujoco_b200 import mjcf, modelpack
    with tempfile.NamedTemporaryFile("w", suffix=".xml", delete=False) as f:
        f.write(xml)
        path = f.name
    try:
        m = mjcf.compile_model(mjcf.XmlHandle(path), fuse_static=False)
    finally:
        os.unlink(path)
    return m, modelpack.pack(m)


class Sim:
    """a bare oracle sim of a compiled model (any library built on the oracle: oracle_binding.load(...).lib)"""

    def __init__(self, o, packed):
        import ctypes
        import numpy as np
        from oracle_binding import _p
        self.lib, self._p = o.lib, _p
        self._keep = [np.ascontiguousarray(packed[0], dtype=np.int32), np.ascontiguousarray(packed[1], dtype=np.float64)]
        a, b = self._keep
        self.sim = ctypes.c_void_p(self.lib.ref_create(_p(a), len(a), _p(b), len(b)))
        assert self.sim.value
        self.nv = self.lib.ref_nv(self.sim)

    def reset(self, q, v):
        import numpy as np
        q, v = np.ascontiguousarray(q, dtype=np.float64), np.ascontiguousarray(v, dtype=np.float64)
        self.lib.ref_reset(self.sim, self._p(q), self._p(v))

    def state(self):
        import numpy as np
        q, v = np.zeros(self.nv), np.zeros(self.nv)
        self.lib.ref_get_state(self.sim, self._p(q), self._p(v))
        return q, v

    def close(self):
        self.lib.ref_destroy(self.sim)
