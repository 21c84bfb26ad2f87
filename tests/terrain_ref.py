"""fp64 reference of the height-field terrain (tests/csrc/terrain_ref.c: the CPU oracle plus mjc_ConvexHField as
include/locosim.h defines it) -- TEST INFRASTRUCTURE ONLY (never imported by the package)."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "csrc", "terrain_ref.c")
DEPS = [SRC, os.path.join(ROOT, "oracle", "locosim_ref.c"), os.path.join(ROOT, "oracle", "locosim_ref.h"),
        os.path.join(ROOT, "include", "locosim_modelpack.h"), os.path.join(ROOT, "include", "locosim_task.h")]
MAXCONPAIR = 50


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def load():
    """the extended oracle library, built on demand"""
    out = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libterrain_ref.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
        tmp = "%s.%d" % (so, os.getpid())
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=gnu11", "-Wall", "-Wno-unused-function", "-fno-fast-math",
                               "-shared", "-o", tmp, SRC, "-lm", "-lpthread"])
        os.replace(tmp, so)
    lib = ctypes.CDLL(so)
    vp, ip, dp = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    lib.reft_create.restype = vp
    lib.reft_create.argtypes = [vp, ip, vp, ip]
    lib.reft_sim.restype = vp
    lib.reft_sim.argtypes = [vp]
    for f, args in [("reft_destroy", [vp]), ("reft_set_origin", [vp, dp, dp]), ("reft_forward", [vp, vp]),
                    ("reft_step", [vp, vp, ip])]:
        getattr(lib, f).restype = None
        getattr(lib, f).argtypes = args
    lib.reft_mpr_calls.restype = ctypes.c_long
    lib.reft_debug_geom.restype = ip
    lib.reft_debug_geom.argtypes = [ip, ip, vp, vp, vp, vp, ip, vp, vp, vp, dp, vp, vp]
    for f, args in [("ref_reset", [vp, vp, vp]), ("ref_get_state", [vp, vp, vp]), ("ref_get_contact", [vp, ip, vp])]:
        getattr(lib, f).restype = None
        getattr(lib, f).argtypes = args
    lib.ref_ncon.restype = ip
    lib.ref_ncon.argtypes = [vp]
    return lib


def debug_geom(lib, hf_data, size4, pos, origin, gtype, gpos, gmat, gsize, margin=0.0):
    """contacts [n, 7] (dist, pos, normal) of one geom against a field; and the number of MPR runs"""
    d = np.ascontiguousarray(hf_data, dtype=np.float64)
    out = np.zeros((MAXCONPAIR, 7))
    nm = ctypes.c_long(0)
    arr = [np.ascontiguousarray(x, dtype=np.float64) for x in (size4, pos, origin, gpos, np.asarray(gmat).reshape(9), gsize)]
    n = lib.reft_debug_geom(d.shape[0], d.shape[1], _p(d), _p(arr[0]), _p(arr[1]), _p(arr[2]), int(gtype), _p(arr[3]),
                            _p(arr[4]), _p(arr[5]), float(margin), _p(out), ctypes.byref(nm))
    return out[:n], nm.value


class Sim:
    """one fp64 sim of a ModelPack with a terrain"""

    def __init__(self, lib, blobs):
        self.lib = lib
        self.ints = np.ascontiguousarray(blobs[0], dtype=np.int32)
        self.reals = np.ascontiguousarray(blobs[1], dtype=np.float64)
        self.h = lib.reft_create(_p(self.ints), len(self.ints), _p(self.reals), len(self.reals))
        assert self.h
        self.sim = lib.reft_sim(self.h)
        self.nv = int(self.ints[3])

    def close(self):
        self.lib.reft_destroy(self.h)

    def set_origin(self, o):
        self.lib.reft_set_origin(self.h, float(o[0]), float(o[1]))

    def reset(self, q, v):
        q, v = np.ascontiguousarray(q, dtype=np.float64), np.ascontiguousarray(v, dtype=np.float64)
        self.lib.ref_reset(self.sim, _p(q), _p(v))

    def state(self):
        q, v = np.zeros(self.nv), np.zeros(self.nv)
        self.lib.ref_get_state(self.sim, _p(q), _p(v))
        return q, v

    def step(self, ctrl, nsub):
        c = np.ascontiguousarray(ctrl, dtype=np.float64)
        self.lib.reft_step(self.h, _p(c), int(nsub))

    def forward(self, ctrl):
        c = np.ascontiguousarray(ctrl, dtype=np.float64)
        self.lib.reft_forward(self.h, _p(c))

    def contacts(self):
        """[ncon, 16] rows of ref_get_contact (dist, pos, normal, geom1, geom2, dim, force[6]) of the last evaluation"""
        n = self.lib.ref_ncon(self.sim)
        out = np.zeros((n, 16))
        for k in range(n):
            row = np.zeros(16)
            self.lib.ref_get_contact(self.sim, k, _p(row))
            out[k] = row
        return out


def ray_hfield(hf, origin, p, v):
    """fp64 mj_rayHfield as include/locosim.h defines it, by brute force: the ray p + x v (world frame) against every top
    triangle of the field (the collision's diagonal), its four sides up to the surface along the edge, and its base.
    Returns (x in units of |v|, outward unit normal) or (-1, zeros)."""
    nrow, ncol = hf.data.shape
    rx, ry, el, bs = hf.size4
    f = np.array([hf.geom_pos[0] - origin[0], hf.geom_pos[1] - origin[1], hf.geom_pos[2]])
    o = np.asarray(p, float) - f
    v = np.asarray(v, float)
    xs = np.linspace(-rx, rx, ncol)
    ys = np.linspace(-ry, ry, nrow)
    Z = hf.data * el
    best, bn = np.inf, np.zeros(3)
    # top triangles: (c, r), (c, r+1), (c+1, r) and (c, r+1), (c+1, r), (c+1, r+1)
    R, C = np.meshgrid(np.arange(nrow - 1), np.arange(ncol - 1), indexing="ij")
    R, C = R.ravel(), C.ravel()
    for tri in (0, 1):
        rr = [R + 1, R, R + 1] if tri else [R, R + 1, R]
        cc = [C, C + 1, C + 1] if tri else [C, C, C + 1]
        P = [np.stack([xs[c], ys[r], Z[r, c]], -1) for r, c in zip(rr, cc)]
        e1, e2 = P[1] - P[0], P[2] - P[0]
        h = np.cross(v, e2)
        det = np.einsum("ij,ij->i", e1, h)
        ok = np.abs(det) > 1e-300
        inv = np.where(ok, 1.0 / np.where(ok, det, 1.0), 0.0)
        s = o - P[0]
        u = inv * np.einsum("ij,ij->i", s, h)
        q = np.cross(s, e1)
        w = inv * (q @ v)
        x = inv * np.einsum("ij,ij->i", e2, q)
        hit = ok & (u >= 0) & (u <= 1) & (w >= 0) & (u + w <= 1) & (x >= 0)
        if hit.any():
            k = np.argmin(np.where(hit, x, np.inf))
            if x[k] < best:
                n = np.cross(e1[k], e2[k])
                best, bn = x[k], n / np.linalg.norm(n) * np.sign(n[2])
    # sides and base
    for ax, sg in ((0, -1), (0, 1), (1, -1), (1, 1)):
        if abs(v[ax]) < 1e-300:
            continue
        plane = sg * (rx if ax == 0 else ry)
        x = (plane - o[ax]) / v[ax]
        if x < 0:
            continue
        q = o + x * v
        oth = 1 - ax
        lim = ry if ax == 0 else rx
        if abs(q[oth]) > lim or q[2] < -bs:
            continue
        edge = Z[:, 0 if sg < 0 else -1] if ax == 0 else Z[0 if sg < 0 else -1, :]
        hz = np.interp(q[oth], ys if ax == 0 else xs, edge)
        if q[2] <= hz and x < best:
            best, bn = x, np.eye(3)[ax] * sg
    if abs(v[2]) > 1e-300:
        x = (-bs - o[2]) / v[2]
        q = o + x * v
        if x >= 0 and abs(q[0]) <= rx and abs(q[1]) <= ry and x < best:
            best, bn = x, np.array([0, 0, -1.0])
    return (best, bn) if np.isfinite(best) else (-1.0, np.zeros(3))
