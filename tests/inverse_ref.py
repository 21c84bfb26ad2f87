"""fp64 reference of the inverse dynamics (tests/csrc/inverse_ref.c: MuJoCo 2.3.7's mj_inverse composed from the CPU
oracle's own stages) and the serial emulation build's entry point for it -- TEST INFRASTRUCTURE ONLY (never imported by the
package)."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_binding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "csrc", "inverse_ref.c")
DEPS = [SRC, os.path.join(ROOT, "tests", "csrc", "applied_forces_ref.c"), os.path.join(ROOT, "oracle", "locosim_ref.c"),
        os.path.join(ROOT, "oracle", "locosim_ref.h"), os.path.join(ROOT, "include", "locosim_modelpack.h"),
        os.path.join(ROOT, "include", "locosim_task.h")]

# The bound of the fp32 engine against this reference, per dof: |got - want| <= C_TOL * 2^-23 * S_d, S_d the first-order
# error scale the reference returns (refinv_inverse). fp32 inverse dynamics is ill-conditioned where contacts are stiff
# (jar is a small difference of large terms), so no fixed atol fits. S_d does not carry the error of the contact geometry
# itself: a convex (MPR) contact's distance is only as accurate as MPR's 1e-6 tolerance, and every contact distance
# carries the rounding of the world positions it is computed from. Measured on the serial core at reset-table states with
# c = 64: at most 0.03 x the bound (UnitreeA1), 1.8 x (Talos), 1.0 x (HumanoidTorque), 0.4 x (UnitreeH1 with arms), 5.6 x
# (Atlas with arms: mesh feet, root 5 m from the origin) and 1.0 x (Talos with arms); hence c = 1024.
C_TOL = 1024.0
EPS32 = 2.0 ** -23
LS_GEOM_BOX, LS_GEOM_MESH = 6, 7          # include/locosim_modelpack.h

_p = oracle_binding._p


def _opt(a):
    return None if a is None else _p(np.ascontiguousarray(a, dtype=np.float64))


def load():
    """Oracle binding of the extended library (the oracle's own entry points are all there too), built on demand."""
    out = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libinverse_ref.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
        # the flags of oracle/Makefile's portable build; built under a temporary name so that a concurrent load never sees
        # a half-written library
        tmp = "%s.%d" % (so, os.getpid())
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=gnu11", "-Wall", "-Wno-unused-function", "-fno-fast-math",
                               "-shared", "-o", tmp, SRC, "-lm", "-lpthread"])
        os.replace(tmp, so)
    o = oracle_binding.load(so)
    lib, vp, ip, dp = o.lib, ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    lib.refinv_forward.restype = ip
    lib.refinv_forward.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.refinv_inverse.restype = dp
    lib.refinv_inverse.argtypes = [vp, vp, vp, vp, vp]
    lib.refinv_cost.restype = dp
    lib.refinv_cost.argtypes = [vp, vp]
    lib.refinv_meaninertia.restype = dp
    lib.refinv_meaninertia.argtypes = [vp]
    lib.refx_nbody.restype = ip
    lib.refx_nbody.argtypes = [vp]
    return o


class InverseSim:
    """One oracle env (model + task blobs, optional user features) for inverse dynamics at given states."""

    def __init__(self, o, model_blobs, task_blobs, user=None, geom_type=None):
        self.geom_type = None if geom_type is None else np.asarray(geom_type)      # (explained(): which contacts are MPR's)
        self.oe = o.env(model_blobs, task_blobs)
        if user is not None:
            self.oe.set_user(user)
        self.lib, self.sim, self.nv = o.lib, self.oe.sim, self.oe.nv
        self.nu = self.lib.ref_nu(self.sim)

    def close(self):
        self.oe.close()

    def forward(self, qpos, qvel, ctrl=None, xfrc=None, qfrc=None):
        """mj_forward at (qpos, qvel) with ctrl [nu] (zeros if None) and applied forces: (qacc, qfrc_actuator, solver
        iterations). Leaves the rows of this state behind for inverse() and cost()."""
        self.oe.set_state(qpos, qvel)
        c = np.zeros(max(self.nu, 1)) if ctrl is None else np.ascontiguousarray(ctrl, dtype=np.float64)
        qacc, act = np.zeros(self.nv), np.zeros(self.nv)
        it = self.lib.refinv_forward(self.sim, _p(c), _opt(xfrc), _opt(qfrc), _p(qacc), _p(act))
        return qacc, act, it

    def inverse(self, qacc):
        """mj_inverse at the state of the last forward(): dict(qfrc [nv], constraint [nv], scale [nv], cost)"""
        qa = np.ascontiguousarray(qacc, dtype=np.float64)
        out, cons, scale = np.zeros(self.nv), np.zeros(self.nv), np.zeros(self.nv)
        cost = self.lib.refinv_inverse(self.sim, _p(qa), _p(out), _p(cons), _p(scale))
        return dict(qfrc=out, constraint=cons, scale=scale, cost=cost)

    def cost(self, qacc):
        """the Newton solver's cost (Gauss + constraint) at qacc over the rows of the last forward()"""
        return self.lib.refinv_cost(self.sim, _p(np.ascontiguousarray(qacc, dtype=np.float64)))

    def at(self, qpos, qvel, qacc):
        """mj_inverse at (qpos, qvel, qacc), with the number of contacts and constraint rows the state gives"""
        self.forward(qpos, qvel)
        r = self.inverse(qacc)
        r["ncon"] = self.lib.ref_ncon(self.sim)
        r["nefc"] = self.lib.ref_nefc(self.sim)
        return r

    def meaninertia(self):
        return self.lib.refinv_meaninertia(self.sim)

    def contact_set_ambiguous(self, qpos, qvel, n_probe=6, seed=0):
        """Whether the contact / constraint set of the state changes under perturbations of qpos / qvel at fp32 resolution
        (relative 4 * 2^-23, at least that absolutely): a contact whose fp64 distance lies within fp32 noise of its
        inclusion margin, where an fp32 engine may include a different set"""
        base = self.at(qpos, qvel, np.zeros(self.nv))
        rng = np.random.RandomState(seed)
        q, v = np.asarray(qpos, dtype=np.float64), np.asarray(qvel, dtype=np.float64)
        for _ in range(n_probe):
            dq = 4 * EPS32 * np.maximum(1.0, np.abs(q)) * rng.choice([-1.0, 1.0], size=q.shape)
            dv = 4 * EPS32 * np.maximum(1.0, np.abs(v)) * rng.choice([-1.0, 1.0], size=v.shape)
            r = self.at(q + dq, v + dv, np.zeros(self.nv))
            if r["ncon"] != base["ncon"] or r["nefc"] != base["nefc"]:
                return True
        return False

    def sensitivity(self, qpos, qvel, qacc, n_probe=6, seed=0):
        """How far the reference's own result [nv] moves when the state is perturbed by the resolution of the contact
        geometry: fp32 resolution (as in contact_set_ambiguous), and at least MPR's 1e-6 tolerance on qpos, to which a
        convex contact's distance is known in either precision. Where a contact is stiff or near a switch, the result moves
        with it and an fp32 engine may land anywhere in that range"""
        base = self.at(qpos, qvel, qacc)["qfrc"]
        rng = np.random.RandomState(seed)
        q, v = np.asarray(qpos, dtype=np.float64), np.asarray(qvel, dtype=np.float64)
        gap = np.zeros(self.nv)
        for _ in range(n_probe):
            dq = np.maximum(4 * EPS32 * np.maximum(1.0, np.abs(q)), 1e-6) * rng.choice([-1.0, 1.0], size=q.shape)
            dv = 4 * EPS32 * np.maximum(1.0, np.abs(v)) * rng.choice([-1.0, 1.0], size=v.shape)
            gap = np.maximum(gap, np.abs(self.at(q + dq, v + dv, qacc)["qfrc"] - base))
        return gap

    def mpr_contact(self, qpos, qvel):
        """whether the state has a contact of a convex pair (box or mesh against a mesh: the MPR narrow phase). fp32 MPR and
        the reference's fp64 MPR each stop at MPR's tolerance, and on deep or near-tied portals they stop on different
        faces: the contact normal and depth then differ by far more than fp32 noise (needs geom_type)"""
        if self.geom_type is None:
            return False
        self.at(qpos, qvel, np.zeros(self.nv))
        for k in range(self.lib.ref_ncon(self.sim)):
            o = np.zeros(16)
            self.lib.ref_get_contact(self.sim, k, _p(o))
            t = {int(self.geom_type[int(o[7])]), int(self.geom_type[int(o[8])])}
            if t <= {LS_GEOM_BOX, LS_GEOM_MESH} and LS_GEOM_MESH in t:
                return True
        return False

    def explained(self, qpos, qvel, qacc, got, want):
        """a result outside the bound that the reference itself explains: the contact set changes at fp32 resolution, an
        MPR contact is present, or the error is within 10x the reference's own jump there"""
        if self.contact_set_ambiguous(qpos, qvel) or self.mpr_contact(qpos, qvel):
            return True
        return bool(np.all(np.abs(np.asarray(got, dtype=np.float64) - want) <= 10 * self.sensitivity(qpos, qvel, qacc)))


def allowed(n):
    """how many of n samples may fail the bound, each explained by the reference: 5 % (rounded down)"""
    return int(0.05 * n)


def within(got, want, scale, c=C_TOL):
    """per dof |got - want| <= c * 2^-23 * scale: (ok, max ratio of error to bound)"""
    bound = c * EPS32 * np.maximum(scale, 1e-30)
    ratio = np.abs(np.asarray(got, dtype=np.float64) - want) / bound
    return bool(np.all(ratio <= 1.0)), float(ratio.max())


def emu_bind(emu):
    """declare emu_inverse(sim, qacc fp64 [nv], out fp32 [nv]) and the other entry points the tests use"""
    vp = ctypes.c_void_p
    emu.emu_inverse.restype = None
    emu.emu_inverse.argtypes = [vp, vp, vp]
    emu.emu_forward.restype = None
    emu.emu_forward.argtypes = [vp, vp]
    emu.emu_get_qacc.restype = None
    emu.emu_get_qacc.argtypes = [vp, vp]
    emu.emu_set_ws.restype = None
    emu.emu_set_ws.argtypes = [vp, vp]
    emu.emu_set_applied.restype = None
    emu.emu_set_applied.argtypes = [vp, vp, vp]
    emu.emu_set_opts.restype = None
    emu.emu_set_opts.argtypes = [vp, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_int]
    emu.emu_iter.restype = ctypes.c_int
    emu.emu_iter.argtypes = [vp]
    return emu
