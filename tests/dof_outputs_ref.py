"""fp64 reference of the per-dof outputs (tests/csrc/dof_outputs_ref.c: the CPU oracle's qfrc_actuator, qfrc_constraint and
qacc, averaged over a control step's sub-steps) and the serial emulation build's entry point for them -- TEST INFRASTRUCTURE
ONLY (never imported by the package)."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_binding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "csrc", "dof_outputs_ref.c")
DEPS = [SRC, os.path.join(ROOT, "oracle", "locosim_ref.c"), os.path.join(ROOT, "oracle", "locosim_ref.h"),
        os.path.join(ROOT, "include", "locosim_modelpack.h"), os.path.join(ROOT, "include", "locosim_task.h")]
DOF_DIM = 3

_p = oracle_binding._p


def load():
    """Oracle binding of the extended library (the oracle's own entry points are all there too), built on demand."""
    out = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libdof_outputs_ref.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
        # the flags of oracle/Makefile's portable build; built under a temporary name so that a concurrent load never sees
        # a half-written library
        tmp = "%s.%d" % (so, os.getpid())
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=gnu11", "-Wall", "-Wno-unused-function", "-fno-fast-math",
                               "-shared", "-o", tmp, SRC, "-lm", "-lpthread"])
        os.replace(tmp, so)
    o = oracle_binding.load(so)
    lib, vp, ip = o.lib, ctypes.c_void_p, ctypes.c_int
    for f, args in [("refdof_add", [vp, vp]), ("refdof_get_forces", [vp, vp, vp]), ("refdof_step", [vp, vp, ip, vp]),
                    ("refdof_env_step", [vp, vp, vp])]:
        getattr(lib, f).restype = None
        getattr(lib, f).argtypes = args
    return o


def now(o, sim):
    """[nv, 3] (qfrc_actuator, qfrc_constraint, qacc) of the last forward evaluation"""
    nv = o.lib.ref_nv(sim)
    out = np.zeros(nv * DOF_DIM)
    o.lib.refdof_add(sim, _p(out))
    return out.reshape(nv, DOF_DIM)


def forces(o, sim):
    """(qfrc_passive, qfrc_actuator) [nv] of the last forward evaluation"""
    nv = o.lib.ref_nv(sim)
    passive, act = np.zeros(nv), np.zeros(nv)
    o.lib.refdof_get_forces(sim, _p(passive), _p(act))
    return passive, act


def step(o, sim, ctrl, nsub):
    """nsub sub-steps of a bare oracle sim at ctrl: the [nv, 3] mean"""
    nv = o.lib.ref_nv(sim)
    out = np.zeros(nv * DOF_DIM)
    c = np.ascontiguousarray(ctrl, dtype=np.float64)
    o.lib.refdof_step(sim, _p(c), int(nsub), _p(out))
    return out.reshape(nv, DOF_DIM)


def env_step(o, oe, action):
    """one control step of oracle env `oe` (physics only): ([nv, 3] mean over its sub-steps, qpos, qvel)"""
    out = np.zeros(oe.nv * DOF_DIM)
    a = np.ascontiguousarray(action, dtype=np.float64)
    o.lib.refdof_env_step(oe.h, _p(a), _p(out))
    q, v = oe.get_state()
    return out.reshape(oe.nv, DOF_DIM), q, v


def sensitivity(o, model_blobs, task_blobs, qpos, qvel, action, ref_dof, warmstart=None, eps=1e-6, n_probe=4, seed=0,
                user=None):
    """How far the ORACLE's own mean moves, per component [3], when its start state is perturbed by `eps` (fp32 resolution):
    the probe of helpers.oracle_step_sensitivity applied to the dof rows. Where a contact switches on or off within the step
    the constraint force is discontinuous, and an fp32 engine may take the other branch."""
    rng = np.random.RandomState(seed)
    gap = np.zeros(DOF_DIM)
    for _ in range(n_probe):
        oe = o.env(model_blobs, task_blobs)
        if user is not None:
            oe.set_user(user)
        oe.set_state(qpos + eps * rng.randn(len(qpos)), qvel + eps * rng.randn(len(qvel)), warmstart)
        d, _, _ = env_step(o, oe, action)
        gap = np.maximum(gap, np.abs(d - ref_dof).max(axis=0))
        oe.close()
    return gap


def emu_bind(emu):
    """declare emu_set_dof(sim, out fp32 [nv, 3] | NULL) on the emulation library"""
    emu.emu_set_dof.restype = None
    emu.emu_set_dof.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    return emu
