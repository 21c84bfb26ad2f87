"""fp64 reference of the body outputs (include/locosim.h locosim_set_body_outputs) from the CPU oracle's own kinematics, and
the serial emulation build's entry point for them -- TEST INFRASTRUCTURE ONLY (never imported by the package).

Positions and orientations are the oracle's xpos / xquat after mj_forward at the state. Velocities are central differences of
those frames along qvel: every in-scope joint is a hinge or a slide (nq = nv), so q + eps qvel is a valid state and
d/dt frame = (frame(q + eps qvel) - frame(q - eps qvel)) / (2 eps); the angular velocity is 2 dq/dt * conj(q) (world frame)."""
import ctypes

import numpy as np

import oracle_binding

_p = oracle_binding._p
BODY_DIM = 13


def quat_mul(a, b):
    w1, x1, y1, z1 = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    w2, x2, y2, z2 = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], axis=-1)


class BodyRef:
    """The oracle's kinematics of one model (oracle_binding.Oracle `o`, compiled model `model`)."""

    def __init__(self, o, model, eps=1e-6):
        from loco_mujoco_b200 import modelpack
        ints, reals = modelpack.pack(model)
        self._keep = (np.ascontiguousarray(ints, dtype=np.int32), np.ascontiguousarray(reals, dtype=np.float64))
        self.lib = o.lib
        self.sim = ctypes.c_void_p(self.lib.ref_create(_p(self._keep[0]), len(self._keep[0]), _p(self._keep[1]),
                                                       len(self._keep[1])))
        assert self.sim.value, "oracle rejected the model"
        self.nv, self.nb, self.eps = model.nv, model.nbody, eps

    def frames(self, q):
        q = np.ascontiguousarray(q, dtype=np.float64)
        self.lib.ref_reset(self.sim, _p(q), None)
        self.lib.ref_forward(self.sim, None)
        xpos, xquat = np.zeros((self.nb, 3)), np.zeros((self.nb, 4))
        self.lib.ref_get_frames(self.sim, _p(xpos), _p(xquat))
        return xpos, xquat

    def __call__(self, q, v):
        """[nbody, 13]: xpos, xquat, angular velocity, linear velocity of the body-frame origin (world frame)."""
        q, v = np.asarray(q, dtype=np.float64), np.asarray(v, dtype=np.float64)
        xp, xq = self.frames(q)
        xp1, xq1 = self.frames(q + self.eps * v)
        xp0, xq0 = self.frames(q - self.eps * v)
        # (q and -q are one rotation: take the neighbours on the side of xq)
        xq1 *= np.sign(np.sum(xq1 * xq, axis=1, keepdims=True) + 1e-300)
        xq0 *= np.sign(np.sum(xq0 * xq, axis=1, keepdims=True) + 1e-300)
        lin = (xp1 - xp0) / (2 * self.eps)
        conj = xq * np.array([1.0, -1, -1, -1])
        ang = 2 * quat_mul((xq1 - xq0) / (2 * self.eps), conj)[:, 1:]
        out = np.concatenate([xp, xq, ang, lin], axis=1)
        out[0] = [0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0]
        return out

    def close(self):
        if self.sim:
            self.lib.ref_destroy(self.sim)
            self.sim = None


def emu_bind(emu):
    emu.emu_body_outputs.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    emu.emu_body_outputs.restype = None


def emu_body(emu, sim, nb):
    out = np.zeros((nb, BODY_DIM), dtype=np.float32)
    emu.emu_body_outputs(sim, _p(out))
    return out


def compare(got, want):
    """Largest error of a [.., nbody, 13] fp32 result against the fp64 reference, each part relative to the magnitudes that
    set its fp32 rounding: positions to 1 + |xpos|max, quaternions (up to sign) to 1, angular velocities to 1 + |w|max,
    linear velocities to 1 + |v|max + |w|max (1 + |xpos|max) (the engine forms them at the CoM and moves them by
    w x (xpos - com), whose terms are as large as |w| |x|). Returns (pos, quat, ang, lin)."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    sp = 1 + np.abs(want[..., 0:3]).max()
    sw = 1 + np.abs(want[..., 7:10]).max()
    sv = 1 + np.abs(want[..., 10:13]).max() + (sw - 1) * sp
    dq = np.minimum(np.abs(got[..., 3:7] - want[..., 3:7]).max(-1), np.abs(got[..., 3:7] + want[..., 3:7]).max(-1))
    return (np.abs(got[..., 0:3] - want[..., 0:3]).max() / sp, dq.max(),
            np.abs(got[..., 7:10] - want[..., 7:10]).max() / sw, np.abs(got[..., 10:13] - want[..., 10:13]).max() / sv)
