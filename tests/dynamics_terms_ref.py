"""fp64 reference of the dynamics terms (include/locosim.h locosim_dynamics_terms: M, qfrc_bias, qfrc_passive, the whole-robot
centre of mass, mj_jacBody at xpos and mj_jacSubtreeCom) from the CPU oracle's own stages (tests/csrc/dynamics_terms_ref.c),
the fp32 error model the engine is held to, and the serial emulation build's entry point -- TEST INFRASTRUCTURE ONLY (never
imported by the package).

M, qfrc_bias and qfrc_passive are the oracle's after a forward evaluation at the state. The centre of mass is
sum m_b xipos_b / sum m_b over the oracle's inertial frames with the model's masses. The Jacobians are central differences
of the oracle's kinematics along each dof (every in-scope joint is a hinge or a slide, nq == nv, so q +- h e_d is a valid
state): the linear rows from xpos (and from the CoM), the angular rows from xquat as vec(q(+h) conj(q(-h))) / h, the
world-frame rotation vector over 2h."""
import ctypes
import copy
import os
import subprocess

import numpy as np

import oracle_binding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "csrc", "dynamics_terms_ref.c")
DEPS = [SRC, os.path.join(ROOT, "oracle", "locosim_ref.c"), os.path.join(ROOT, "oracle", "locosim_ref.h"),
        os.path.join(ROOT, "include", "locosim_modelpack.h"), os.path.join(ROOT, "include", "locosim_task.h")]
EPS32 = 2.0 ** -23
TERMS = ("M", "bias", "passive", "com", "jac", "jac_com")

# fp32 error model. Every term is a sum of products of fp32 quantities; to first order its error is bounded by
# 2^-23 times the sum of the absolute values of those products, times the number of roundings on the way (the kinematic
# chain's depth, a few per level), which the constant C_TOL stands for:
#   M_ij       S = sum_k |cdof_j|_k (|crb_i| |cdof_i|)_k + |armature_i|     (crb_factor's products, in absolute values)
#   bias_d     S = sum_k |cdof_d|_k sum_{b in subtree(d)} (|I_b| |a_b| + |v_b| x* |I_b v_b|)_k     (passive_bias's RNE)
#   passive_d  S = |k_d| (|q_d| + |q_spring,d|) + |b_d qvel_d|
#   mass       S = sum_b m_b
# and everything built from lever arms (the com-frame quantities above, the CoM, the Jacobians' linear rows) also carries
# the rounding of the world positions the arms are differences of: an absolute eps * P per position, P = max_b |xpos_b|
# (the robot's distance from the world origin, in metres). Those scales are multiplied by W = 1 + P (lever arms of the
# in-scope robots are O(1 m)), and for the CoM and the Jacobians (values of O(1) in m or m/rad):
#   com (x, y, z)          S = W
#   jac rows 0-2 (angular)  S = 1
#   jac rows 3-5, jac_com   S = W
# The scales of M and bias are the sums of the absolute values of the oracle's own products on the magnitudes of their
# factors (tests/csrc/dynamics_terms_ref.c). C_TOL: with C = 256 the largest error was 0.24 x the bound on the serial core
# (20 reset-table states with perturbed velocities per configuration; M of the 31-dof models) and 0.03 x on an H100 (80
# rollout states per kernel family; M of Atlas with arms).
C_TOL = 256.0

_p = oracle_binding._p


def load():
    """Oracle binding of the extended library (the oracle's own entry points are all there too), built on demand."""
    out = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libdynamics_terms_ref.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
        # the flags of oracle/Makefile's portable build; built under a temporary name so that a concurrent load never sees
        # a half-written library
        tmp = "%s.%d" % (so, os.getpid())
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=gnu11", "-Wall", "-Wno-unused-function", "-fno-fast-math",
                               "-shared", "-o", tmp, SRC, "-lm", "-lpthread"])
        os.replace(tmp, so)
    o = oracle_binding.load(so)
    lib, vp = o.lib, ctypes.c_void_p
    lib.refdyn_terms.restype = None
    lib.refdyn_terms.argtypes = [vp] * 9
    lib.refdyn_frames.restype = None
    lib.refdyn_frames.argtypes = [vp] * 5
    lib.refdyn_nbody.restype = ctypes.c_int
    lib.refdyn_nbody.argtypes = [vp]
    return o


def quat_mul(a, b):
    w1, x1, y1, z1 = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    w2, x2, y2, z2 = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], axis=-1)


def model_with_pool_row(m, row):
    """A copy of compiled model m carrying the parameters of one parameter-pool row (domain_randomization.POOL_FIELDS)."""
    from loco_mujoco_b200.domain_randomization import POOL_FIELDS
    m = copy.deepcopy(m)
    off = 0
    for field, _, _ in POOL_FIELDS:
        shape = np.shape(getattr(m, field))
        n = int(np.prod(shape))
        setattr(m, field, np.asarray(row[off:off + n], dtype=np.float64).reshape(shape))
        off += n
    m.stat_meaninertia = float(row[off])
    return m


class DynRef:
    """The oracle's dynamics terms of one compiled model (oracle_binding.Oracle `o` of load())."""

    def __init__(self, o, model, h=1e-6):
        from loco_mujoco_b200 import modelpack
        ints, reals = modelpack.pack(model)
        self._keep = (np.ascontiguousarray(ints, dtype=np.int32), np.ascontiguousarray(reals, dtype=np.float64))
        self.lib = o.lib
        self.sim = ctypes.c_void_p(self.lib.ref_create(_p(self._keep[0]), len(self._keep[0]), _p(self._keep[1]),
                                                       len(self._keep[1])))
        assert self.sim.value, "oracle rejected the model"
        self.nv, self.nb, self.h = model.nv, model.nbody, h
        assert self.lib.refdyn_nbody(self.sim) == self.nb
        self.mass = np.asarray(model.body_mass, dtype=np.float64)
        self.stiffness = np.asarray(model.jnt_stiffness, dtype=np.float64)
        self.damping = np.asarray(model.dof_damping, dtype=np.float64)
        self.spring = np.asarray(model.qpos_spring, dtype=np.float64)

    def close(self):
        if self.sim is not None:
            self.lib.ref_destroy(self.sim)
            self.sim = None

    def frames(self, q):
        """(xpos [nb, 3], xquat [nb, 4], xipos [nb, 3]) of the oracle's kinematics at q"""
        xp, xq, xi = np.zeros((self.nb, 3)), np.zeros((self.nb, 4)), np.zeros((self.nb, 3))
        self.lib.refdyn_frames(self.sim, _p(np.ascontiguousarray(q, dtype=np.float64)), _p(xp), _p(xq), _p(xi))
        return xp, xq, xi

    def com_at(self, q):
        _, _, xi = self.frames(q)
        return (self.mass[:, None] * xi).sum(0) / self.mass.sum()

    def terms(self, q, v, jac=True):
        """dict of the six terms in the engine's layout (fp64) and their error scales ("s_" + name)"""
        q = np.asarray(q, dtype=np.float64)
        v = np.asarray(v, dtype=np.float64)
        nv, nb = self.nv, self.nb
        M, bias, passive, com = np.zeros((nv, nv)), np.zeros(nv), np.zeros(nv), np.zeros(4)
        sM, sbias = np.zeros((nv, nv)), np.zeros(nv)
        self.lib.refdyn_terms(self.sim, _p(np.ascontiguousarray(q)), _p(np.ascontiguousarray(v)), _p(M), _p(bias),
                              _p(passive), _p(com), _p(sM), _p(sbias))
        xpos, _, _ = self.frames(q)
        P = float(np.abs(xpos).max())
        W = 1.0 + P
        r = dict(M=M, bias=bias, passive=passive, com=com, s_M=W * sM, s_bias=W * sbias,
                 s_passive=np.abs(self.stiffness) * (np.abs(q) + np.abs(self.spring)) + np.abs(self.damping * v),
                 s_com=np.array([W, W, W, self.mass.sum()]), P=P)
        if jac:
            J, Jc = np.zeros((nb, 6, nv)), np.zeros((3, nv))
            for d in range(nv):
                e = np.zeros(nv)
                e[d] = self.h
                xp1, xq1, xi1 = self.frames(q + e)
                xp0, xq0, xi0 = self.frames(q - e)
                dq = quat_mul(xq1, xq0 * np.array([1.0, -1.0, -1.0, -1.0]))
                dq *= np.sign(dq[:, :1]) + (dq[:, :1] == 0)
                J[:, :3, d] = dq[:, 1:] / self.h
                J[:, 3:, d] = (xp1 - xp0) / (2 * self.h)
                m = self.mass[:, None]
                Jc[:, d] = ((m * xi1).sum(0) - (m * xi0).sum(0)) / (2 * self.h * self.mass.sum())
            J[0] = 0.0
            sJ = np.empty((nb, 6, nv))
            sJ[:, :3], sJ[:, 3:] = 1.0, W
            r.update(jac=J, jac_com=Jc, s_jac=sJ, s_jac_com=np.full((3, nv), W))
        return r


def within(got, want, scale, c=C_TOL):
    """|got - want| <= c 2^-23 scale entrywise: (ok, max ratio of error to bound)"""
    bound = c * EPS32 * np.maximum(np.asarray(scale, dtype=np.float64), 1e-30)
    ratio = np.abs(np.asarray(got, dtype=np.float64) - want) / bound
    return bool(np.all(ratio <= 1.0)), float(ratio.max())


def check(got, ref, c=C_TOL):
    """{term: max ratio of error to bound} of the terms in `got` (a dict keyed as TERMS) against DynRef.terms() `ref`;
    asserts every term within its bound"""
    out = {}
    for k, x in got.items():
        if x is None:
            continue
        ok, ratio = within(x, ref[k], ref["s_" + k], c)
        assert ok, (k, ratio, np.unravel_index(np.argmax(np.abs(np.asarray(x, np.float64) - ref[k])), np.shape(x)))
        out[k] = ratio
    return out


def emu_bind(emu):
    """declare emu_dynamics_terms(sim, M, bias, passive, com, jac, jac_com) (fp32 outputs, each may be NULL)"""
    emu.emu_dynamics_terms.restype = None
    emu.emu_dynamics_terms.argtypes = [ctypes.c_void_p] * 7
    return emu


def emu_terms(emu, s, nv, nb, q, v):
    """the serial core's six terms at (q, v) of emulated env s (model parameters), fp32, in the engine's layout"""
    emu.emu_reset(s, _p(np.ascontiguousarray(q, dtype=np.float64)), _p(np.ascontiguousarray(v, dtype=np.float64)))
    out = dict(M=np.full((nv, nv), np.nan, np.float32), bias=np.full(nv, np.nan, np.float32),
               passive=np.full(nv, np.nan, np.float32), com=np.full(4, np.nan, np.float32),
               jac=np.full((nb, 6, nv), np.nan, np.float32), jac_com=np.full((3, nv), np.nan, np.float32))
    emu.emu_dynamics_terms(s, *[out[k].ctypes.data_as(ctypes.c_void_p) for k in TERMS])
    return out
