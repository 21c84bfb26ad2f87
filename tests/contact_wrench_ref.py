"""fp64 reference of the per-body contact wrenches (tests/csrc/contact_wrench_ref.c: the CPU oracle plus the sum of
mj_contactForce over each body's contacts) and the serial emulation build's entry point for them -- TEST INFRASTRUCTURE ONLY
(never imported by the package)."""
import ctypes
import os
import subprocess

import numpy as np

import oracle_binding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "csrc", "contact_wrench_ref.c")
DEPS = [SRC, os.path.join(ROOT, "oracle", "locosim_ref.c"), os.path.join(ROOT, "oracle", "locosim_ref.h"),
        os.path.join(ROOT, "include", "locosim_modelpack.h"), os.path.join(ROOT, "include", "locosim_task.h")]
CONTACT_DIM = 6

_p = oracle_binding._p


def load():
    """Oracle binding of the extended library (the oracle's own entry points are all there too), built on demand."""
    out = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libcontact_wrench_ref.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
        # the flags of oracle/Makefile's portable build; built under a temporary name so that a concurrent load never sees
        # a half-written library
        tmp = "%s.%d" % (so, os.getpid())
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=gnu11", "-Wall", "-Wno-unused-function", "-fno-fast-math",
                               "-shared", "-o", tmp, SRC, "-lm", "-lpthread"])
        os.replace(tmp, so)
    o = oracle_binding.load(so)
    lib, vp, ip = o.lib, ctypes.c_void_p, ctypes.c_int
    lib.refcw_nbody.restype = ip
    lib.refcw_nbody.argtypes = [vp]
    for f, args in [("refcw_get_contact", [vp, ip, vp]), ("refcw_add_wrench", [vp, vp]), ("refcw_env_step", [vp, vp, vp]),
                    ("refcw_step", [vp, vp, ip, vp])]:
        getattr(lib, f).restype = None
        getattr(lib, f).argtypes = args
    return o


def contacts(o, sim):
    """the contact list of the last forward evaluation: [ncon, 22] rows of refcw_get_contact (dist, pos, frame rows n t1 t2,
    geom1, geom2, dim, contact-frame force f[6])"""
    n = o.lib.ref_ncon(sim)
    out = np.zeros((n, 22))
    for k in range(n):
        row = np.zeros(22)
        o.lib.refcw_get_contact(sim, k, _p(row))
        out[k] = row
    return out


def wrench_now(o, sim):
    """[nb, 6] per-body contact wrench of the last forward evaluation"""
    nb = o.lib.refcw_nbody(sim)
    w = np.zeros(nb * CONTACT_DIM)
    o.lib.refcw_add_wrench(sim, _p(w))
    return w.reshape(nb, CONTACT_DIM)


def env_step(o, oe, action):
    """one control step of oracle env `oe` (physics only): ([nb, 6] mean wrench over its sub-steps, qpos, qvel)"""
    nb = o.lib.refcw_nbody(oe.sim)
    w = np.zeros(nb * CONTACT_DIM)
    a = np.ascontiguousarray(action, dtype=np.float64)
    o.lib.refcw_env_step(oe.h, _p(a), _p(w))
    q, v = oe.get_state()
    return w.reshape(nb, CONTACT_DIM), q, v


def step(o, sim, ctrl, nsub):
    """nsub sub-steps of a bare oracle sim at ctrl: the [nb, 6] mean wrench"""
    nb = o.lib.refcw_nbody(sim)
    w = np.zeros(nb * CONTACT_DIM)
    c = np.ascontiguousarray(ctrl, dtype=np.float64)
    o.lib.refcw_step(sim, _p(c), int(nsub), _p(w))
    return w.reshape(nb, CONTACT_DIM)


def sensitivity(o, model_blobs, task_blobs, qpos, qvel, action, ref_wrench, warmstart=None, eps=1e-6, n_probe=4, seed=0,
                user=None):
    """How far the ORACLE's own mean wrench moves when its start state is perturbed by `eps` (fp32 resolution): the probe of
    helpers.oracle_step_sensitivity applied to the wrench rows. Where a contact switches on or off within the step the
    wrench is discontinuous, and an fp32 engine may take the other branch."""
    rng = np.random.RandomState(seed)
    gap = 0.0
    for _ in range(n_probe):
        oe = o.env(model_blobs, task_blobs)
        if user is not None:
            oe.set_user(user)
        oe.set_state(qpos + eps * rng.randn(len(qpos)), qvel + eps * rng.randn(len(qvel)), warmstart)
        w, _, _ = env_step(o, oe, action)
        gap = max(gap, float(np.abs(w - ref_wrench).max()))
        oe.close()
    return gap


def emu_bind(emu):
    """declare emu_set_contact(sim, wrench fp32 [nb, 6] | NULL) on the emulation library"""
    emu.emu_set_contact.restype = None
    emu.emu_set_contact.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    return emu
