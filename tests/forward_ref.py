"""fp64 reference of the forward dynamics outputs (tests/csrc/forward_ref.c: MuJoCo 2.3.7's mj_forward + mj_rnePostConstraint
on the CPU oracle's own stages) and the serial emulation build's entry point for them -- TEST INFRASTRUCTURE ONLY (never
imported by the package)."""
import ctypes
import os
import subprocess

import numpy as np

import inverse_ref
import oracle_binding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "csrc", "forward_ref.c")
DEPS = [SRC] + inverse_ref.DEPS
DOF_DIM, BODY_ACC_DIM, CONTACT_DIM = 3, 6, 6          # include/locosim.h
OUTPUTS = ("dof", "body_acc", "cfrc_int", "cfrc_ext")

# The bound of the fp32 engine against this reference, per output and component: |got - want| <= REL * max(1, max |want|)
# over the rows of the state (one scale per output and component group: the dof output per column, the body rows per
# angular / linear half). Every output is a linear map of qacc and the constraint forces at the state, so it carries their
# error: the fp32 Newton solver stops at a scaled gradient of 1e-5, not at the fp64 solution, and stiff contacts amplify
# the difference in qacc into the contact forces. Measured on the serial core at reset-table states under random actions:
# at most 8e-5 of the magnitude (Atlas with arms: mesh feet, 5 m from the origin); hence 2e-3.
# Where a contact is within fp32 noise of switching, the reference's own result jumps: there the error must stay within 10x
# that jump (ForwardSim.sensitivity).
REL = 2e-3

_p = oracle_binding._p


def _opt(a):
    return None if a is None else _p(np.ascontiguousarray(a, dtype=np.float64))


def load():
    """Oracle binding of the extended library (the oracle's and the inverse reference's entry points are all there too)"""
    out = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libforward_ref.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
        tmp = "%s.%d" % (so, os.getpid())
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=gnu11", "-Wall", "-Wno-unused-function", "-fno-fast-math",
                               "-shared", "-o", tmp, SRC, "-lm", "-lpthread"])
        os.replace(tmp, so)
    return _bind(so)


def _bind(so):
    o = oracle_binding.load(so)
    lib, vp, ip, dp = o.lib, ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    lib.refinv_forward.restype = ip
    lib.refinv_forward.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.refinv_inverse.restype = dp
    lib.refinv_inverse.argtypes = [vp, vp, vp, vp, vp]
    lib.refx_nbody.restype = ip
    lib.refx_nbody.argtypes = [vp]
    lib.reffwd_forward.restype = ip
    lib.reffwd_forward.argtypes = [vp] * 9
    lib.reffwd_frames.restype = None
    lib.reffwd_frames.argtypes = [vp] * 6
    lib.reffwd_kin.restype = None
    lib.reffwd_kin.argtypes = [vp] * 5
    return o


class ForwardSim:
    """One oracle env (model + task blobs, optional user features) for forward dynamics at given states"""

    def __init__(self, o, model_blobs, task_blobs=None, user=None):
        """an oracle env of (model, task) blobs, or with task_blobs None a bare oracle sim of the model blobs alone"""
        if task_blobs is None:
            from position_mode import Sim
            self.oe = Sim(o, model_blobs)
            self._set = self.oe.reset
        else:
            self.oe = o.env(model_blobs, task_blobs)
            if user is not None:
                self.oe.set_user(user)
            self._set = self.oe.set_state
        self.lib, self.sim, self.nv = o.lib, self.oe.sim, self.oe.nv
        self.nu = self.lib.ref_nu(self.sim)
        self.nb = self.lib.refx_nbody(self.sim)

    def close(self):
        self.oe.close()

    def forward(self, qpos, qvel, ctrl=None, xfrc=None, qfrc=None):
        """mj_forward + mj_rnePostConstraint at (qpos, qvel) with ctrl [nu] (zeros if None) and applied forces (xfrc
        [nb, 6] force then torque at xipos, qfrc [nv]): dict of the four outputs in the engine's layout, MuJoCo's own
        spatial cacc / cfrc_int / cfrc_ext ("raw" [nb, 3, 6], about the subtree CoM), the solver's iterations ("iter"), and
        the frames of the evaluation (cdof [nv, 6], cinert [nb, 10], xipos / subtree_com [nb, 3], passive [nv])"""
        self._set(np.asarray(qpos, dtype=np.float64), np.asarray(qvel, dtype=np.float64))
        c = np.zeros(max(self.nu, 1)) if ctrl is None else np.ascontiguousarray(ctrl, dtype=np.float64)
        nv, nb = self.nv, self.nb
        r = dict(dof=np.zeros((nv, DOF_DIM)), body_acc=np.zeros((nb, BODY_ACC_DIM)), cfrc_int=np.zeros((nb, CONTACT_DIM)),
                 cfrc_ext=np.zeros((nb, CONTACT_DIM)), raw=np.zeros((nb, 3, 6)))
        r["iter"] = self.lib.reffwd_forward(self.sim, _p(c), _opt(xfrc), _opt(qfrc), _p(r["dof"]), _p(r["body_acc"]),
                                            _p(r["cfrc_int"]), _p(r["cfrc_ext"]), _p(r["raw"]))
        fr = dict(cdof=np.zeros((nv, 6)), cinert=np.zeros((nb, 10)), xipos=np.zeros((nb, 3)), subtree_com=np.zeros((nb, 3)),
                  passive=np.zeros(nv))
        self.lib.reffwd_frames(self.sim, _p(fr["cdof"]), _p(fr["cinert"]), _p(fr["xipos"]), _p(fr["subtree_com"]),
                               _p(fr["passive"]))
        r.update(fr)
        return r

    def kin(self, qpos):
        """(xpos [nb, 3], cdof [nv, 6], subtree_com [nb, 3]) of the kinematics alone at qpos"""
        xpos, cdof, com = np.zeros((self.nb, 3)), np.zeros((self.nv, 6)), np.zeros((self.nb, 3))
        self.lib.reffwd_kin(self.sim, _p(np.ascontiguousarray(qpos, dtype=np.float64)), _p(xpos), _p(cdof), _p(com))
        return xpos, cdof, com

    def sensitivity(self, qpos, qvel, ctrl, want, n_probe=6, seed=0, eps=1e-6):
        """per output, the largest move of the reference's own result [same shape] under perturbations of the state by
        fp32 resolution (relative 4 * 2^-23, at least `eps` on qpos: MPR's tolerance), where a contact switches"""
        rng = np.random.RandomState(seed)
        q, v = np.asarray(qpos, dtype=np.float64), np.asarray(qvel, dtype=np.float64)
        gap = {k: np.zeros_like(want[k]) for k in OUTPUTS}
        e32 = 4 * 2.0 ** -23
        for _ in range(n_probe):
            dq = np.maximum(e32 * np.maximum(1.0, np.abs(q)), eps) * rng.choice([-1.0, 1.0], size=q.shape)
            dv = e32 * np.maximum(1.0, np.abs(v)) * rng.choice([-1.0, 1.0], size=v.shape)
            r = self.forward(q + dq, v + dv, ctrl)
            for k in OUTPUTS:
                gap[k] = np.maximum(gap[k], np.abs(r[k] - want[k]))
        return gap


def groups(x, name):
    """the component groups of an output [rows, cols] that share one scale: the dof output per column, the body outputs
    per angular / linear (or force / torque) half"""
    if name == "dof":
        return [x[:, c] for c in range(x.shape[1])]
    return [x[:, :3], x[:, 3:]]


def within(got, want, name, gap=None, rel=REL):
    """per group: |got - want| <= rel * max(1, max |want|) (or < 10x the reference's own jump `gap` there): (ok, worst
    ratio of error to bound)"""
    ok, worst = True, 0.0
    gg = groups(np.zeros_like(want) if gap is None else gap, name)
    for g, w, j in zip(groups(np.asarray(got, dtype=np.float64), name), groups(want, name), gg):
        tol = rel * max(1.0, float(np.abs(w).max()))
        err = np.abs(g - w)
        worst = max(worst, float(err.max()) / tol)
        if not np.all((err <= tol) | (err < 10 * j)):
            ok = False
    return ok, worst


def emu_bind(emu):
    """declare emu_forward_outputs(sim, ctrl fp64 [nu], dof, body_acc, cfrc_int, cfrc_ext fp32 or NULL) and the entry points
    the tests use with it"""
    vp = ctypes.c_void_p
    inverse_ref.emu_bind(emu)
    emu.emu_forward_outputs.restype = None
    emu.emu_forward_outputs.argtypes = [vp] * 6
    return emu


def emu_forward(emu, s, nv, nb, q, v, ctrl, ws=None, which=OUTPUTS):
    """the serial core's forward outputs at (q, v) from warm start ws (zeros if None): {name: fp32 array}"""
    emu.emu_reset(s, _p(np.ascontiguousarray(q, dtype=np.float64)), _p(np.ascontiguousarray(v, dtype=np.float64)))
    emu.emu_set_ws(s, _p(np.zeros(nv) if ws is None else np.ascontiguousarray(ws, dtype=np.float64)))
    shapes = dict(dof=(nv, DOF_DIM), body_acc=(nb, BODY_ACC_DIM), cfrc_int=(nb, CONTACT_DIM), cfrc_ext=(nb, CONTACT_DIM))
    out = {k: np.full(shapes[k], np.nan, dtype=np.float32) for k in which}
    c = np.ascontiguousarray(ctrl if len(ctrl) else np.zeros(1), dtype=np.float64)
    emu.emu_forward_outputs(s, _p(c), *[_p(out[k]) if k in out else None for k in OUTPUTS])
    return out
