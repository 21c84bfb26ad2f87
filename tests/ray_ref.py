"""fp64 reference of ray casting (include/locosim.h locosim_ray, MuJoCo 2.3.7's mj_ray) and the serial build's entry point
for it -- TEST INFRASTRUCTURE ONLY (never imported by the package).

Geom frames come from the CPU oracle's kinematics (body_outputs_ref.BodyRef) and the compiled geom_pos / geom_quat. The
primitives are MuJoCo's engine_ray.c written out in numpy fp64. A mesh geom is cast against the convex hull of its vertices
by a different algorithm from the device's GJK ray cast: slab clipping against the facet planes of
scipy.spatial.ConvexHull(verts).equations.

A ray is AMBIGUOUS when which geom it hits is decided by less than the fp32 error: its geom changes when every geom is grown
or shrunk by `delta`, or when its start point moves by `delta` along any axis, or when the runner-up hit lies within
`delta` of the first. Its normal is only compared where it is INTERIOR to a face: the same (to 1e-3) under those moves."""
import ctypes

import numpy as np

from body_outputs_ref import quat_mul
import oracle_binding

_p = oracle_binding._p
PLANE, SPHERE, CAPSULE, ELLIPSOID, CYLINDER, BOX, MESH = 0, 2, 3, 4, 5, 6, 7
WORLD, BODY, HEADING, TRACK = 0, 1, 2, 3
STATIC, DYNAMIC, PER_ENV = 1, 2, 4


def quat_mat(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


class Scene:
    """The geoms of one compiled model at one state, fp64 world frames, and what a query selects of them."""

    def __init__(self, model, xpos, xquat):
        from scipy.spatial import ConvexHull
        self.m, self.xpos, self.xquat = model, np.asarray(xpos, dtype=np.float64), np.asarray(xquat, dtype=np.float64)
        m = model
        self.pos, self.mat, self.hull = [], [], []
        dofmask = np.zeros(m.nbody, dtype=bool)
        for j in range(m.nv):
            dofmask[m.jnt_bodyid[j]] = True
        moving = np.zeros(m.nbody, dtype=bool)
        for b in range(1, m.nbody):
            moving[b] = dofmask[b] or moving[m.body_parentid[b]]
        self.static = ~moving[np.asarray(m.geom_bodyid)]
        for g in range(m.ngeom):
            b = m.geom_bodyid[g]
            self.pos.append(self.xpos[b] + quat_mat(self.xquat[b]) @ np.asarray(m.geom_pos[g], dtype=np.float64))
            self.mat.append(quat_mat(quat_mul(self.xquat[b], np.asarray(m.geom_quat[g], dtype=np.float64))))
            if m.geom_type[g] == MESH:
                a, n = m.geom_meshadr[g], m.geom_meshnum[g]
                v = np.asarray(m.mesh_vert, dtype=np.float64).reshape(-1, 3)[a:a + n]
                self.hull.append(ConvexHull(v).equations)
            else:
                self.hull.append(None)

    def to_world(self, frame, fb, pnt, vec):
        pnt, vec = np.asarray(pnt, dtype=np.float64), np.asarray(vec, dtype=np.float64)
        if frame == WORLD:
            return pnt, vec
        x = self.xpos[fb]
        if frame == BODY:
            R = quat_mat(self.xquat[fb])
        elif frame == HEADING:
            f = quat_mat(self.xquat[fb])[:, 0]
            h = np.hypot(f[0], f[1])
            c, s = (f[0] / h, f[1] / h) if h > 1e-6 else (1.0, 0.0)
            R = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])
        else:
            R = np.eye(3)
        return x + pnt @ R.T, vec @ R.T

    def cast(self, p, v, exclude=-1, sel=STATIC | DYNAMIC, grow=0.0):
        """per ray (p, v [n, 3], world): (x [n], geom [n], normal [n, 3], runner-up x [n]) with every geom grown by `grow`"""
        n = len(p)
        X = np.full((n, self.m.ngeom), np.inf)
        N = np.zeros((n, self.m.ngeom, 3))
        for g in range(self.m.ngeom):
            ok = (STATIC if self.static[g] else DYNAMIC) & sel
            if not ok or self.m.geom_bodyid[g] == exclude:
                continue
            R = self.mat[g]
            lp, lv = (p - self.pos[g]) @ R, v @ R
            x, ln = _geom(self.m.geom_type[g], np.asarray(self.m.geom_size[g], dtype=np.float64), self.hull[g], lp, lv, grow)
            hit = x >= 0
            X[hit, g] = x[hit]
            N[:, g] = ln @ R.T
        order = np.argsort(X, axis=1)
        first, second = order[:, 0], order[:, 1] if self.m.ngeom > 1 else order[:, 0]
        rows = np.arange(n)
        x = X[rows, first]
        geom = np.where(np.isfinite(x), first, -1)
        nrm = N[rows, first]
        nrm = nrm / np.maximum(np.linalg.norm(nrm, axis=1, keepdims=True), 1e-300)
        nrm[geom < 0] = 0
        x2 = X[rows, second] if self.m.ngeom > 1 else np.full(n, np.inf)
        return np.where(geom >= 0, x, -1.0), geom, nrm, x2

    def classify(self, p, v, delta, **kw):
        """(x, geom, normal, ambiguous [n] bool, face_interior [n] bool) of world rays p, v (see the module docstring)"""
        x, geom, nrm, x2 = self.cast(p, v, **kw)
        vl = np.linalg.norm(v, axis=1)
        amb = np.isfinite(x2) & (geom >= 0) & ((x2 - x) * vl < 2 * delta)
        interior = np.ones(len(p), dtype=bool)
        moves = [dict(grow=delta), dict(grow=-delta)] + [dict(shift=s * delta * e) for e in np.eye(3) for s in (1, -1)]
        for mv in moves:
            pp = p + mv.get("shift", 0)
            x1, g1, n1, _ = self.cast(pp, v, grow=mv.get("grow", 0.0), **kw)
            amb |= g1 != geom
            interior &= (g1 == geom) & (np.abs(n1 - nrm).max(axis=1) < 1e-3)
        return x, geom, nrm, amb, interior & ~amb


def _quad(p, v, r2):
    """roots of |p + x v|^2 = r2 (rows), nan where none"""
    a = (v * v).sum(1)
    b = (p * v).sum(1)
    c = (p * p).sum(1) - r2
    with np.errstate(invalid="ignore", divide="ignore"):
        d = b * b - a * c
        s = np.sqrt(np.where(d >= 0, d, np.nan))
        return (-b - s) / a, (-b + s) / a


def _first(x0, x1):
    return np.where(x0 >= 0, x0, np.where(x1 >= 0, x1, -1.0))


def _geom(t, s, eq, lp, lv, grow):
    n = len(lp)
    ln = np.zeros((n, 3))
    x = np.full(n, -1.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        if t == PLANE:
            xx = -(lp[:, 2] - grow) / lv[:, 2]
            q = lp + xx[:, None] * lv
            ok = (lv[:, 2] < 0) & (xx >= 0) & ((s[0] <= 0) | (np.abs(q[:, 0]) <= s[0] + grow)) & \
                ((s[1] <= 0) | (np.abs(q[:, 1]) <= s[1] + grow))
            x = np.where(ok, xx, -1.0)
            ln[:] = [0, 0, 1]
        elif t in (SPHERE, ELLIPSOID):
            sz = np.full(3, s[0]) if t == SPHERE else s
            sz = sz + grow
            x = _first(*_quad(lp / sz, lv / sz, 1.0))
            q = lp + np.maximum(x, 0)[:, None] * lv
            ln = q / sz ** 2
        elif t in (CAPSULE, CYLINDER):
            r, h = s[0] + grow, s[1] + (grow if t == CYLINDER else 0.0)
            cand = []
            x0, x1 = _quad(lp[:, :2], lv[:, :2], r * r)
            for xx in (x0, x1):
                q = lp + xx[:, None] * lv
                cand.append((np.where((xx >= 0) & (np.abs(q[:, 2]) <= h), xx, np.nan),
                             np.concatenate([q[:, :2], np.zeros((n, 1))], axis=1)))
            for side in (-1, 1):
                if t == CAPSULE:
                    c = np.array([0, 0, side * h])
                    for xx in _quad(lp - c, lv, r * r):
                        q = lp + xx[:, None] * lv
                        cand.append((np.where((xx >= 0) & (side * q[:, 2] >= h), xx, np.nan), q - c))
                else:
                    xx = (side * h - lp[:, 2]) / lv[:, 2]
                    q = lp + xx[:, None] * lv
                    cand.append((np.where((xx >= 0) & ((q[:, :2] ** 2).sum(1) <= r * r), xx, np.nan),
                                 np.tile([0, 0, side], (n, 1)).astype(float)))
            x, ln = _best(cand, n)
        elif t == BOX:
            sz = s + grow
            cand = []
            for i in range(3):
                for side in (-1, 1):
                    xx = (side * sz[i] - lp[:, i]) / lv[:, i]
                    q = lp + xx[:, None] * lv
                    j, k = [a for a in range(3) if a != i]
                    ok = (xx >= 0) & (np.abs(q[:, j]) <= sz[j]) & (np.abs(q[:, k]) <= sz[k])
                    nn = np.zeros((n, 3))
                    nn[:, i] = side
                    cand.append((np.where(ok, xx, np.nan), nn))
            x, ln = _best(cand, n)
        elif t == MESH:
            nrm, off = eq[:, :3], eq[:, 3] - grow
            a = lp @ nrm.T + off            # > 0: outside the facet's plane
            b = lv @ nrm.T
            tt = -a / b
            enter = np.where(b < 0, tt, -np.inf)
            leave = np.where(b > 0, tt, np.inf)
            miss = ((b == 0) & (a > 0)).any(1)
            te, tl = enter.max(1), leave.min(1)
            ie, il = enter.argmax(1), leave.argmin(1)
            hit = ~miss & (te <= tl) & (tl >= 0)
            x = np.where(hit, np.where(te >= 0, te, tl), -1.0)
            ln = np.where((te >= 0)[:, None], nrm[ie], nrm[il])
    x = np.where(np.isfinite(x) & (x >= 0), x, -1.0)
    return x, ln


def _best(cand, n):
    xs = np.stack([c[0] for c in cand], axis=1)
    xs = np.where(np.isnan(xs), np.inf, xs)
    k = xs.argmin(1)
    x = xs[np.arange(n), k]
    ln = np.stack([c[1] for c in cand], axis=1)[np.arange(n), k]
    return np.where(np.isfinite(x), x, -1.0), ln


def emu_bind(emu):
    emu.emu_ray.restype = None
    emu.emu_ray.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                            ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]


def emu_ray(emu, sim, pnt, vec, frame=WORLD, fb=0, exclude=-1, sel=STATIC | DYNAMIC):
    """the serial build's cast of the emulated env's current state: (dist fp32 [n], geom int32 [n], normal fp32 [n, 3])"""
    pnt = np.ascontiguousarray(pnt, dtype=np.float32)
    vec = np.ascontiguousarray(vec, dtype=np.float32)
    n = len(pnt)
    dist, geom, nrm = np.zeros(n, np.float32), np.zeros(n, np.int32), np.zeros((n, 3), np.float32)
    emu.emu_ray(sim, _p(pnt), _p(vec), n, frame, fb, exclude, sel, _p(dist), _p(geom), _p(nrm))
    return dist, geom, nrm


def scale(p, x, v, rb):
    """the magnitude that sets a hit's fp32 rounding: |pnt| + x |vec| + the hit geom's bounding radius"""
    return np.linalg.norm(p, axis=1) + np.maximum(x, 0) * np.linalg.norm(v, axis=1) + rb


DIST_TOL = 2e-5      # about 170 fp32 epsilons


def dist_ok(got, x, p, v, rb, nrm):
    """the fp32 error model of a hit's distance: |x_fp32 - x_fp64| |vec| <= DIST_TOL * scale / max(|cos|, 1e-3), with cos
    the cosine between the ray and the normal (an error across the surface moves a grazing hit along the ray by 1 / cos)"""
    vl = np.linalg.norm(v, axis=1)
    cos = np.abs((nrm * v).sum(1)) / np.maximum(vl, 1e-300)
    return np.abs(got - x) * vl <= DIST_TOL * scale(p, x, v, rb) / np.maximum(cos, 1e-3)
