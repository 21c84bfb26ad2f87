"""The capsule-hull test of sphere | capsule | cylinder pairs (locosim_core.cuh capsule_hulls_apart, pair flag 4).

A convex pair that passes the bounding spheres and the box test becomes an MPR job. For a cylinder against a capsule or a
sphere the box bounds the cylinder poorly, so the engine also tests the distance between the geoms' axis segments. These
tests check that the test rejects only pairs that are really apart (brute-force geometry in fp64), that a seeded UnitreeA1
rollout of the serial emulation build is the same with the test on and off (LOCOSIM_DEBUG bit 32 turns it off), and, on the
GPU, that 4096 UnitreeA1 envs step to the same bits with it on and off."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, golden, make_env

SPHERE, CAPSULE, CYLINDER = 2, 3, 5
NO_HULL_TEST = 32          # LOCOSIM_DEBUG bit


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def hull(emu):
    f = emu.emu_capsule_hulls_apart
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p] * 2 + [ctypes.c_float]
    emu.emu_set_debug.argtypes = [ctypes.c_int]
    emu.emu_set_debug.restype = None
    emu.emu_mpr_stat.argtypes = [ctypes.c_int]
    emu.emu_mpr_stat.restype = ctypes.c_long
    return emu


def _rot(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _point_cylinder(p, r, h):
    """distance of points p [..., 3] (cylinder frame) to the solid cylinder of radius r and half length h"""
    dr = np.maximum(np.hypot(p[..., 0], p[..., 1]) - r, 0.0)
    dz = np.maximum(np.abs(p[..., 2]) - h, 0.0)
    return np.hypot(dr, dz)


def _segment_cylinder(a, b, r, h):
    """distance of the segment a-b (cylinder frame) to the solid cylinder: convex along the segment, so a dense scan and a
    golden-section refinement around its best sample give the minimum"""
    s = np.linspace(0.0, 1.0, 2049)
    d = _point_cylinder(a + s[:, None] * (b - a), r, h)
    k = int(np.argmin(d))
    lo, hi = s[max(k - 1, 0)], s[min(k + 1, len(s) - 1)]
    f = lambda t: float(_point_cylinder(a + t * (b - a), r, h))
    g = (np.sqrt(5) - 1) / 2
    for _ in range(80):
        c, e = hi - g * (hi - lo), lo + g * (hi - lo)
        if f(c) < f(e):
            hi = e
        else:
            lo = c
    return min(float(d.min()), f(0.5 * (lo + hi)))


def _pose_cases(rng, n):
    """(other type, other size, other pos, other frame, cylinder size, cylinder pos, cylinder frame): random poses with
    the other geom placed near the cylinder, including parallel, coaxial cap-on and rim-touching ones"""
    for k in range(n):
        cs = np.array([rng.uniform(0.01, 0.06), rng.uniform(0.005, 0.08), 0.0], np.float32)
        cp = rng.uniform(-3, 3, 3).astype(np.float32)
        cm = _rot(rng)
        t = SPHERE if k % 3 == 0 else CAPSULE
        os_ = np.array([rng.uniform(0.01, 0.05), rng.uniform(0.01, 0.12) if t == CAPSULE else 0.0, 0.0], np.float32)
        kind = k % 5
        if kind == 0:            # parallel, side by side
            om = cm.copy()
            off = cm @ np.array([1.0, 0.0, rng.uniform(-2, 2) * cs[1]]) * (cs[0] + os_[0] + rng.uniform(-0.01, 0.01))
        elif kind == 1:          # coaxial, on a cap
            om = cm.copy() if rng.random() < 0.5 else cm @ _rot(rng)
            off = cm[:, 2] * (cs[1] + os_[0] + os_[1] * abs(om[:, 2] @ cm[:, 2]) + rng.uniform(-0.01, 0.01))
        elif kind == 2:          # at the rim
            om = _rot(rng)
            ang = rng.uniform(0, 2 * np.pi)
            rim = cm @ np.array([cs[0] * np.cos(ang), cs[0] * np.sin(ang), cs[1]])
            dirn = rng.normal(size=3)
            dirn /= np.linalg.norm(dirn)
            off = rim + dirn * (os_[0] + rng.uniform(-0.005, 0.02))
        else:                    # anywhere near
            om = _rot(rng)
            off = rng.normal(size=3) * (cs[0] + cs[1] + os_[0] + os_[1])
        yield t, os_, (cp + off).astype(np.float32), om.astype(np.float32), cs, cp, cm.astype(np.float32)


def test_capsule_hull_test_rejects_only_separated_pairs(hull):
    rng = np.random.default_rng(7)
    rejected = kept = 0
    for t, os_, op, om, cs, cp, cm in _pose_cases(rng, 3000):
        margin = np.float32(rng.choice([0.0, 0.001, 0.01]))
        om32, cm32 = np.ascontiguousarray(om.reshape(9)), np.ascontiguousarray(cm.reshape(9))
        apart = hull.emu_capsule_hulls_apart(t, _p(op), _p(om32), _p(os_), CYLINDER, _p(cp), _p(cm32),
                                             _p(cs.copy()), margin)
        # brute force in fp64, in the cylinder's frame as MPR sees it (the fp32 frame, the fp32 positions)
        cm64, om64 = cm.astype(np.float64), om.astype(np.float64)
        h = 0.0 if t == SPHERE else float(os_[1])
        a = cm64.T @ (op.astype(np.float64) - h * om64[:, 2] - cp)
        b = cm64.T @ (op.astype(np.float64) + h * om64[:, 2] - cp)
        gap = _segment_cylinder(a, b, float(cs[0]), float(cs[1])) - float(os_[0]) - float(margin)
        if apart:
            rejected += 1
            assert gap > 0, "an intersecting pair was rejected (gap %.3e)" % gap
        else:
            kept += 1
        # the hull is tight along the side: well-separated side-by-side pairs are rejected
        if gap > 1e-4 and abs(a[2]) <= cs[1] and abs(b[2]) <= cs[1]:
            assert apart, "a pair %.3e apart beside the cylinder was kept" % gap
    print("capsule-hull test: %d of %d poses rejected" % (rejected, rejected + kept))
    assert rejected > 300 and kept > 300


def _support(t, size, pos, frame, n):
    """fp64 support function h(n) = max over the geom of n . x (sphere, capsule, solid cylinder; frame columns = axes)"""
    z = frame[:, 2]
    nz = float(n @ z)
    if t == SPHERE:
        return float(n @ pos) + size[0]
    if t == CAPSULE:
        return float(n @ pos) + size[1] * abs(nz) + size[0]
    return float(n @ pos) + size[1] * abs(nz) + size[0] * np.sqrt(max(0.0, 1.0 - nz * nz))


def _separation(t1, s1, p1, f1, t2, s2, p2, f2, rng):
    """a lower bound of the distance of two convex geoms (fp64): the best separation -h2(-n) - h1(n) over directions n,
    started from the closest points of the axis segments (dense scan) and refined by random perturbations"""
    h1 = 0.0 if t1 == SPHERE else s1[1]
    h2 = 0.0 if t2 == SPHERE else s2[1]
    s = np.linspace(-1.0, 1.0, 401)
    a = p1[None, :] + (s * h1)[:, None] * f1[:, 2][None, :]
    b = p2[None, :] + (s * h2)[:, None] * f2[:, 2][None, :]
    dd = np.linalg.norm(a[:, None, :] - b[None, :, :], axis=2)
    i, j = np.unravel_index(np.argmin(dd), dd.shape)
    n = b[j] - a[i]
    n = n / max(np.linalg.norm(n), 1e-300)
    sep = lambda n: -_support(t2, s2, p2, f2, -n) - _support(t1, s1, p1, f1, n)
    best = sep(n)
    for scale in (1e-1, 1e-2, 1e-3, 1e-4):
        for _ in range(60):
            m = n + rng.normal(size=3) * scale
            m /= np.linalg.norm(m)
            v = sep(m)
            if v > best:
                best, n = v, m
    return best


def test_capsule_hull_test_of_cylinder_pairs_in_both_orders(hull):
    """pair flag 4 is set for any axial pair against a cylinder, in either order, cylinder vs cylinder included: every
    rejected pose must be separated (an fp64 separating direction proves it), and swapping the geoms changes nothing"""
    rng = np.random.default_rng(11)
    rejected = 0
    n = 1500
    for k in range(n):
        cs = np.array([rng.uniform(0.01, 0.06), rng.uniform(0.005, 0.08), 0.0], np.float32)
        cm = _rot(rng).astype(np.float32)
        cp = rng.uniform(-3, 3, 3).astype(np.float32)
        t = (SPHERE, CAPSULE, CYLINDER)[k % 3]
        os_ = np.array([rng.uniform(0.01, 0.05), 0.0 if t == SPHERE else rng.uniform(0.01, 0.1), 0.0], np.float32)
        kind = k % 4
        if kind == 0:        # parallel or antiparallel within a fraction of a degree, side by side
            om = cm @ _rot_small(rng, rng.choice([0.0, 1e-3, 5e-3, 2e-2]))
            if rng.random() < 0.5:
                om = om @ np.diag([1.0, -1.0, -1.0])
            off = cm @ np.array([1.0, 0.0, rng.uniform(-1.5, 1.5) * cs[1]]) * (cs[0] + os_[0] + rng.uniform(-2e-3, 2e-3))
        elif kind == 1:      # crossing at a right angle, near touching
            om = cm @ np.array([[1.0, 0, 0], [0, 0, -1], [0, 1, 0]])
            off = cm @ np.array([cs[0] + os_[0] + rng.uniform(-2e-3, 2e-3), 0.0, rng.uniform(-1, 1) * cs[1]])
        elif kind == 2:      # end on end
            om = cm @ _rot_small(rng, rng.uniform(0, 0.5))
            off = cm[:, 2] * (cs[1] + os_[1] + os_[0] * (t == SPHERE) + rng.uniform(-2e-3, 5e-3))
        else:
            om = _rot(rng)
            off = rng.normal(size=3) * (cs[0] + cs[1] + os_[0] + os_[1])
        om = om.astype(np.float32)
        op = (cp + off).astype(np.float32)
        margin = np.float32(rng.choice([0.0, 0.001, 0.01]))
        om9, cm9 = np.ascontiguousarray(om.reshape(9)), np.ascontiguousarray(cm.reshape(9))
        fwd = hull.emu_capsule_hulls_apart(t, _p(op), _p(om9), _p(os_), CYLINDER, _p(cp), _p(cm9), _p(cs), margin)
        rev = hull.emu_capsule_hulls_apart(CYLINDER, _p(cp), _p(cm9), _p(cs), t, _p(op), _p(om9), _p(os_), margin)
        assert fwd == rev, (k, fwd, rev)
        if fwd:
            rejected += 1
            sep = _separation(t, os_.astype(np.float64), op.astype(np.float64), om.astype(np.float64), CYLINDER,
                              cs.astype(np.float64), cp.astype(np.float64), cm.astype(np.float64), rng)
            assert sep > float(margin), "pose %d rejected, but no direction separates it by the margin (%.3e)" % (k, sep)
    print("cylinder pairs, both orders: %d of %d poses rejected" % (rejected, n))
    assert 150 < rejected < n - 150


def _rot_small(rng, angle):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def test_capsule_hull_test_of_touching_and_crossing_segments(hull):
    eye = np.eye(3, dtype=np.float32).reshape(9)
    side = np.array([[1, 0, 0], [0, 0, -1], [0, 1, 0]], np.float32).reshape(9)    # z axis along -y
    cs = np.array([0.03, 0.05, 0], np.float32)
    os_ = np.array([0.02, 0.1, 0], np.float32)
    z = np.zeros(3, np.float32)
    for frame in (eye, side):
        for dx, apart in ((0.05, 0), (0.0501, 1), (0.0499, 0), (0.0, 0)):
            op = np.array([dx, 0.0, 0.0], np.float32)
            got = hull.emu_capsule_hulls_apart(CAPSULE, _p(op), _p(frame.copy()), _p(os_.copy()), CYLINDER, _p(z.copy()),
                                               _p(eye.copy()), _p(cs.copy()), np.float32(0.0))
            assert got == apart, (frame.reshape(3, 3)[:, 2], dx, got)


def _rollout(emu, task, steps, seed):
    from loco_mujoco_b200 import modelpack
    env = make_env(task)
    m, spec, g = env._model, env.task_spec(), golden(task)
    ints, reals = modelpack.pack(m)
    sim = emu.emu_create(_p(ints), len(ints), _p(reals), len(reals))
    assert sim
    q0, v0 = np.zeros(m.nq), np.zeros(m.nq)
    for t, i, val in zip(spec.obs_src_type, spec.obs_src_idx, g[0]):
        if t == 0:
            q0[i] = val
        elif t == 1:
            v0[i] = val
    rng = np.random.default_rng(seed)
    q, v, ws = np.zeros(m.nq), np.zeros(m.nq), np.zeros(m.nq)
    out = []
    emu.emu_reset(sim, _p(q0), _p(v0))
    for k in range(steps):
        if k % 60 == 0 and k:
            emu.emu_reset(sim, _p(q0), _p(v0))
        ctrl = np.zeros(m.nu)
        ctrl[spec.act_idx] = rng.uniform(-1, 1, len(spec.act_idx)) * spec.act_delta + spec.act_mean
        emu.emu_step(sim, _p(ctrl), spec.n_substeps)
        emu.emu_get_state(sim, _p(q), _p(v))
        emu.emu_get_ws(sim, _p(ws))
        out.append(np.concatenate([q, v, ws, [emu.emu_ncon(sim)]]))
    emu.emu_destroy(sim)
    return np.array(out)


def test_emulated_rollout_is_unchanged_by_the_capsule_hull_test(hull, bundled_only):
    emu = hull
    emu.emu_get_ws.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    emu.emu_ncon.argtypes = [ctypes.c_void_p]
    emu.emu_ncon.restype = ctypes.c_int
    runs, jobs, mpr = {}, {}, {}
    try:
        for dbg in (NO_HULL_TEST, 0):
            emu.emu_set_debug(dbg)
            j0, c0 = emu.emu_mpr_stat(7), emu.emu_mpr_stat(2)
            runs[dbg] = _rollout(emu, "UnitreeA1.simple", 240, seed=3)
            jobs[dbg], mpr[dbg] = emu.emu_mpr_stat(7) - j0, emu.emu_mpr_stat(2) - c0
    finally:
        emu.emu_set_debug(0)
    print("UnitreeA1.simple, 240 steps: convex jobs %d without the capsule-hull test, %d with it; MPR runs %d -> %d"
          % (jobs[NO_HULL_TEST], jobs[0], mpr[NO_HULL_TEST], mpr[0]))
    assert np.array_equal(runs[0], runs[NO_HULL_TEST])
    assert jobs[NO_HULL_TEST] > 0 and jobs[0] < 0.5 * jobs[NO_HULL_TEST]


_GPU_SCRIPT = r"""
import os, sys, torch
sys.path.insert(0, sys.argv[1])
os.environ["LOCO_MUJOCO_B200_FORCE_BUNDLED"] = "1"
from loco_mujoco_b200 import LocoEnv
env = LocoEnv.make("UnitreeA1.simple", num_envs=4096, seed=5)
eng = env._get_engine()
g = torch.Generator(device=eng.device).manual_seed(11)
acts = torch.rand((50, eng.n_envs, eng.action_dim), device=eng.device, generator=g) * 2 - 1
eng.reset()
outs = []
for k in range(50):
    obs, rew, done, nxt = eng.step(acts[k])
    outs += [obs.clone(), rew.clone(), done.clone(), nxt.clone()]
    if k % 10 == 9:
        outs += [x.clone() for x in eng.get_state()]           # qpos, qvel, warm start
torch.cuda.synchronize()
torch.save({"outs": [o.cpu() for o in outs], "info": str(eng.launch_info())}, sys.argv[2])
"""


@pytest.mark.gpu
def test_gpu_steps_are_unchanged_by_the_capsule_hull_test(tmp_path):
    import torch
    script = tmp_path / "run.py"
    script.write_text(_GPU_SCRIPT)
    res = {}
    for dbg in (NO_HULL_TEST, 0):
        out = tmp_path / ("run%d.pt" % dbg)
        env = dict(os.environ, LOCOSIM_DEBUG=str(dbg))
        subprocess.check_call([sys.executable, str(script), ROOT, str(out)], env=env)
        res[dbg] = torch.load(out)
    a, b = res[0], res[NO_HULL_TEST]
    print(a["info"])
    assert len(a["outs"]) == len(b["outs"]) == 50 * 4 + 5 * 3
    for k, (x, y) in enumerate(zip(a["outs"], b["outs"])):
        assert torch.equal(x, y), k
