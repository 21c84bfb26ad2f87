"""fp64 reference of applied forces (tests/csrc/applied_forces_ref.c: the CPU oracle plus xfrc_applied / qfrc_applied) and
the serial emulation build's setter for them -- TEST INFRASTRUCTURE ONLY (never imported by the package)."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_binding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "csrc", "applied_forces_ref.c")
DEPS = [SRC, os.path.join(ROOT, "oracle", "locosim_ref.c"), os.path.join(ROOT, "oracle", "locosim_ref.h"),
        os.path.join(ROOT, "include", "locosim_modelpack.h"), os.path.join(ROOT, "include", "locosim_task.h")]

_p = oracle_binding._p


def _opt(a):
    return None if a is None else _p(a)


def load():
    """Oracle binding of the extended library (the oracle's own entry points are all there too), built on demand."""
    out = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libapplied_forces_ref.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
        # the flags of oracle/Makefile's portable build
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=gnu11", "-Wall", "-Wno-unused-function", "-fno-fast-math",
                               "-shared", "-o", so, SRC, "-lm", "-lpthread"])
    o = oracle_binding.load(so)
    lib, vp, ip = o.lib, ctypes.c_void_p, ctypes.c_int
    lib.refx_nbody.restype = ip
    lib.refx_nbody.argtypes = [vp]
    for f, args in [("refx_forward", [vp, vp, vp, vp]), ("refx_step", [vp, vp, ip, vp, vp]),
                    ("refx_env_step", [vp, vp, vp, vp]), ("refx_get_bodies", [vp, vp, vp])]:
        getattr(lib, f).restype = None
        getattr(lib, f).argtypes = args
    return o


def _f64(a, shape):
    return None if a is None else np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(shape))


class AppliedSim:
    """One oracle env (model + task blobs) with applied forces: xfrc [nb, 6] (force, torque; world frame, at the body CoM),
    qfrc [nv]; either None = not applied."""

    def __init__(self, o, model_blobs, task_blobs, user=None):
        self.oe = o.env(model_blobs, task_blobs)
        if user is not None:
            self.oe.set_user(user)
        self.lib, self.sim, self.nv = o.lib, self.oe.sim, self.oe.nv
        self.nb = self.lib.refx_nbody(self.sim)

    def reset_to(self, traj_no, step_no):
        return self.oe.reset_to(traj_no, step_no)

    def set_state(self, qpos, qvel):
        self.oe.set_state(qpos, qvel)

    def get_state(self):
        return self.oe.get_state()

    def env_step(self, action, xfrc=None, qfrc=None):
        """one control step (physics only); returns (qpos, qvel)"""
        a = np.ascontiguousarray(action, dtype=np.float64)
        x, q = _f64(xfrc, (self.nb, 6)), _f64(qfrc, (self.nv,))
        self.lib.refx_env_step(self.oe.h, _p(a), _opt(x), _opt(q))
        return self.get_state()

    def step(self, ctrl, nsub, xfrc=None, qfrc=None):
        c = np.ascontiguousarray(ctrl, dtype=np.float64)
        x, q = _f64(xfrc, (self.nb, 6)), _f64(qfrc, (self.nv,))
        self.lib.refx_step(self.sim, _p(c), int(nsub), _opt(x), _opt(q))
        return self.get_state()

    def forward(self, qpos, qvel, ctrl, xfrc=None, qfrc=None):
        """mj_forward at (qpos, qvel, ctrl) with the forces: dict of qfrc_smooth, qacc_smooth, M, xipos [nb, 3], xmat [nb, 3, 3]"""
        self.set_state(qpos, qvel)
        c = np.ascontiguousarray(ctrl, dtype=np.float64)
        x, q = _f64(xfrc, (self.nb, 6)), _f64(qfrc, (self.nv,))
        self.lib.refx_forward(self.sim, _p(c), _opt(x), _opt(q))
        nv, nb = self.nv, self.nb
        qs, qa, M = np.zeros(nv), np.zeros(nv), np.zeros((nv, nv))
        xipos, xmat = np.zeros((nb, 3)), np.zeros((nb, 3, 3))
        self.lib.ref_get_smooth(self.sim, _p(qs), _p(qa))
        self.lib.ref_get_M(self.sim, _p(M))
        self.lib.refx_get_bodies(self.sim, _p(xipos), _p(xmat))
        return dict(qfrc_smooth=qs, qacc_smooth=qa, M=M, xipos=xipos, xmat=xmat)

    def close(self):
        self.oe.close()


def emu_bind_applied(emu):
    """declare emu_set_applied(sim, xfrc fp32 [nb, 6] | NULL, qfrc fp32 [nv] | NULL) on the emulation library"""
    emu.emu_set_applied.restype = None
    emu.emu_set_applied.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return emu
