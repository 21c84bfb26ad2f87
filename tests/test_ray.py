"""Ray casting (MuJoCo's mj_ray, include/locosim.h locosim_ray; LocoEnv.ray_cast / camera / render) without a GPU: the
header constants, the Python layer's refusals, the serial build of the CUDA core on closed-form scenes of every geom type and
against the fp64 reference (tests/ray_ref.py) at oracle rollout states of every bundled model, and the camera's ray set."""
import os
import subprocess
import tempfile
import types

import numpy as np
import pytest

import ray_ref as rr
from body_outputs_ref import BodyRef
from full_body import make_variant
from helpers import ROOT, oracle_env
from position_mode import compile_xml, make_position

p = rr._p


class _Emu:
    """the serial core of a compiled model at one state"""

    def __init__(self, emu, packed):
        rr.emu_bind(emu)
        self.emu = emu
        self.ints = np.ascontiguousarray(packed[0], dtype=np.int32)
        self.reals = np.ascontiguousarray(packed[1], dtype=np.float64)
        self.s = emu.emu_create(p(self.ints), len(self.ints), p(self.reals), len(self.reals))
        assert self.s

    def cast(self, q, pnt, vec, **kw):
        q = np.ascontiguousarray(q, dtype=np.float64)
        self.emu.emu_reset(self.s, p(q), p(np.zeros_like(q)))
        return rr.emu_ray(self.emu, self.s, pnt, vec, **kw)

    def close(self):
        self.emu.emu_destroy(self.s)


SCENE = """
<mujoco model="shapes">
  <option timestep="0.002"/>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 1"/>
    <geom name="tile" type="plane" size="0.5 0.25 1" pos="0 0 -1"/>
    <body name="b" pos="0 0 0">
      <joint name="z" type="slide" axis="0 0 1"/>
      <geom name="sphere" type="sphere" size="0.2" pos="0 0 1"/>
      <geom name="capsule" type="capsule" size="0.1 0.3" pos="2 0 1"/>
      <geom name="ellipsoid" type="ellipsoid" size="0.1 0.2 0.3" pos="4 0 1"/>
      <geom name="cylinder" type="cylinder" size="0.15 0.25" pos="6 0 1"/>
      <geom name="box" type="box" size="0.1 0.2 0.3" pos="8 0 1"/>
    </body>
  </worldbody>
</mujoco>
"""


@pytest.fixture(scope="module")
def shapes(emu):
    m, packed = compile_xml(SCENE)
    e = _Emu(emu, packed)
    yield m, e
    e.close()


def _down(x, y, z=3.0):
    return np.array([[x, y, z]]), np.array([[0.0, 0.0, -1.0]])


@pytest.mark.parametrize("name, x, top", [("sphere", 0, 1.2), ("capsule", 2, 1.4), ("ellipsoid", 4, 1.3),
                                          ("cylinder", 6, 1.25), ("box", 8, 1.3)])
def test_known_distance_and_normal_from_above(shapes, name, x, top):
    m, e = shapes
    d, g, n = e.cast([0.0], *_down(x, 0))
    assert g[0] == m.geom_names.index(name)
    assert abs(d[0] - (3 - top)) < 1e-6 and np.allclose(n[0], [0, 0, 1], atol=1e-6)


@pytest.mark.parametrize("name, x, side", [("sphere", 0, 0.2), ("capsule", 2, 0.1), ("ellipsoid", 4, 0.1),
                                           ("cylinder", 6, 0.15), ("box", 8, 0.1)])
def test_known_distance_and_normal_from_the_side(shapes, name, x, side):
    """a ray along +x at the geom's centre height, from 1 m before its centre, with |vec| = 2: dist in units of |vec|"""
    m, e = shapes
    d, g, n = e.cast([0.0], [[x - 1.0, 0, 1]], [[2.0, 0, 0]], sel=rr.DYNAMIC)
    assert g[0] == m.geom_names.index(name)
    assert abs(d[0] - (1 - side) / 2) < 1e-6 and np.allclose(n[0], [-1, 0, 0], atol=1e-6)


def test_a_ray_that_starts_inside_reports_its_exit(shapes):
    m, e = shapes
    for name, x, exit_ in (("sphere", 0, 0.2), ("capsule", 2, 0.1), ("ellipsoid", 4, 0.1), ("cylinder", 6, 0.15),
                           ("box", 8, 0.1)):
        d, g, n = e.cast([0.0], [[x, 0, 1]], [[1.0, 0, 0]], sel=rr.DYNAMIC)
        assert g[0] == m.geom_names.index(name) and abs(d[0] - exit_) < 1e-6, name
        assert np.allclose(n[0], [1, 0, 0], atol=1e-6)


def test_the_floor_is_one_sided_and_finite_planes_keep_their_size(shapes):
    m, e = shapes
    floor, tile = m.geom_names.index("floor"), m.geom_names.index("tile")
    # parallel to the floor, and from below it, misses; from above it hits at the height
    d, g, _ = e.cast([0.0], [[10, 0, 0.5], [10, 0, -0.5], [10, 0, 0.5]], [[1, 0, 0], [0, 0, 1.0], [0, 0, -1.0]])
    assert list(g) == [-1, -1, floor] and d[0] == -1 and d[1] == -1 and abs(d[2] - 0.5) < 1e-7
    # the tile at z = -1 is 0.5 x 0.25: below the floor, only reached with the floor excluded (body 0 excludes both)
    d, g, _ = e.cast([0.0], [[0.4, 0.2, -0.5], [0.6, 0.0, -0.5], [0.0, 0.3, -0.5]], [[0, 0, -1.0]] * 3)
    assert list(g) == [tile, -1, -1] and abs(d[0] - 0.5) < 1e-7


def test_exclude_body_static_and_dynamic_select_their_geoms(shapes):
    m, e = shapes
    pnt, vec = _down(0, 0)
    assert e.cast([0.0], pnt, vec)[1][0] == m.geom_names.index("sphere")
    assert e.cast([0.0], pnt, vec, sel=rr.STATIC)[1][0] == m.geom_names.index("floor")
    assert e.cast([0.0], pnt, vec, exclude=1)[1][0] == m.geom_names.index("floor")
    assert e.cast([0.0], pnt, vec, sel=rr.DYNAMIC, exclude=1)[1][0] == -1
    assert e.cast([0.0], pnt, vec, sel=0)[1][0] == -1
    # the body moves with its slide joint
    d, g, _ = e.cast([0.5], pnt, vec)
    assert g[0] == m.geom_names.index("sphere") and abs(d[0] - (3 - 1.7)) < 1e-6
    # a zero vec hits nothing
    assert e.cast([0.0], pnt, [[0.0, 0, 0]])[1][0] == -1


CUBE = """
<mujoco model="cube">
  <asset><mesh name="cube" file="{obj}"/></asset>
  <worldbody>
    <body name="b" pos="0 0 1" euler="10 20 30">
      <joint name="z" type="slide" axis="0 0 1"/>
      <geom name="hull" type="mesh" mesh="cube"/>
      <body name="c">
        <geom name="box" type="box" size="0.5 0.5 0.5"/>
      </body>
    </body>
  </worldbody>
</mujoco>
"""


def test_a_unit_cube_hull_matches_the_box_routine(emu):
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "cube.obj")
        with open(obj, "w") as f:
            for v in np.array(np.meshgrid([-.5, .5], [-.5, .5], [-.5, .5], indexing="ij")).reshape(3, -1).T:
                f.write("v %g %g %g\n" % tuple(v))
            for face in ((1, 3, 4, 2), (5, 6, 8, 7), (1, 2, 6, 5), (3, 7, 8, 4), (1, 5, 7, 3), (2, 4, 8, 6)):
                f.write("f %d %d %d\nf %d %d %d\n" % (face[0], face[1], face[2], face[0], face[2], face[3]))
        m, packed = compile_xml(CUBE.format(obj=obj))
    e = _Emu(emu, packed)
    rng = np.random.RandomState(0)
    pnt = rng.uniform(-2, 2, (400, 3)) + [0, 0, 1]
    vec = (rng.uniform(-0.6, 0.6, (400, 3)) + [0, 0, 1]) - pnt
    pnt[:40] = rng.uniform(-0.3, 0.3, (40, 3)) + [0, 0, 1]                 # starts inside: the exit point
    hull_body, box_body = m.geom_bodyid[m.geom_names.index("hull")], m.geom_bodyid[m.geom_names.index("box")]
    dh, gh, nh = e.cast([0.0], pnt, vec, exclude=box_body)
    db, gb, nb = e.cast([0.0], pnt, vec, exclude=hull_body)
    assert np.array_equal(gh >= 0, gb >= 0) and (gh >= 0).sum() > 300
    hit = gh >= 0
    assert np.abs(dh[hit] - db[hit]).max() * np.linalg.norm(vec, axis=1).max() < 2e-5
    assert np.abs(nh[hit] - nb[hit]).max() < 2e-3
    e.close()


# ---------------------------------------------------------------------------------------------------------------------
# every bundled model against the fp64 reference at oracle rollout states
# ---------------------------------------------------------------------------------------------------------------------
MODELS = ["UnitreeA1.simple", "UnitreeA1.simple+position", "Talos.walk", "UnitreeH1.walk", "HumanoidTorque.run",
          "Atlas.walk", "UnitreeG1.walk", "HumanoidTorque4Ages.walk.2", "Atlas.walk+arms", "Talos.walk+arms"]


def _make(task, **kw):
    if task.endswith("+position"):
        return make_position(task[:-len("+position")], **kw)
    return make_variant(task, **kw)


def oracle_states(oracle, env, n, steps, seed):
    """n states of the oracle's random-action rollouts from reset-table rows"""
    spec = env.task_spec()
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        oe = oracle_env(oracle, env)
        oe.reset_to(rng.randint(spec.table.shape[0]), rng.randint(spec.table.shape[1]))
        for _ in range(steps):
            oe.step(rng.uniform(-1, 1, env._model.nu))
        out.append(oe.get_state()[0])
        oe.close()
    return out


def random_rays(rng, n, frame):
    """rays of a query frame that mostly meet the robot or the floor: from about 1.5 m around the frame's origin (world:
    around the robot's start position) towards points near it"""
    pnt = rng.normal(0, 1.0, (n, 3))
    pnt[:, 2] = np.abs(pnt[:, 2]) + 0.3
    aim = rng.normal(0, 0.3, (n, 3))
    if frame == rr.WORLD:
        pnt[:, 2] += 0.5
        aim[:, 2] += 0.6
    vec = (aim - pnt) * rng.uniform(0.3, 3.0, (n, 1))
    return pnt, vec


def compare(model, scene, p, v, x, geom, nrm, rb_of):
    """(ambiguous count, largest scaled distance error, largest normal error) of one cast against the reference"""
    wp, wv = p, v
    delta = 1e-5 * (1 + np.linalg.norm(wp, axis=1).max() + np.linalg.norm(wv, axis=1).max())
    xr, gr, nr, amb, interior = scene.classify(wp, wv, delta)
    ok = ~amb
    assert np.array_equal(geom[ok], gr[ok]), (np.nonzero(geom[ok] != gr[ok])[0][:5])
    hit = ok & (gr >= 0)
    dist_ok = rr.dist_ok(x[hit], xr[hit], wp[hit], wv[hit], rb_of[gr[hit]], nr[hit])
    nerr = np.abs(nrm[interior & hit] - nr[interior & hit]).max(initial=0)
    return int(amb.sum()), dist_ok.all(), nerr


@pytest.mark.parametrize("task", MODELS)
def test_serial_core_matches_the_fp64_reference(emu, oracle, bundled_only, task):
    """Random rays in all four frames at 6 oracle rollout states: geom ids agree outside the ambiguous set (bounded at 3 %
    of the rays), distances within rr.dist_ok's fp32 error model, normals to 2e-3 where the hit is interior to a face"""
    from loco_mujoco_b200 import modelpack
    env = _make(task, num_envs=4)
    m = env._model
    e = _Emu(emu, [np.asarray(x) for x in modelpack.pack(m)])
    body = BodyRef(oracle, m)
    rng = np.random.RandomState(3)
    rb = np.asarray(m.geom_rbound, dtype=np.float64)
    n_amb = n_all = n_hit = 0
    for q in oracle_states(oracle, env, 6, 5, 7):
        xpos, xquat = body.frames(q)
        scene = rr.Scene(m, xpos, xquat)
        for frame in (rr.WORLD, rr.BODY, rr.HEADING, rr.TRACK):
            fb = 0 if frame == rr.WORLD else int(rng.randint(1, m.nbody))
            pnt, vec = random_rays(rng, 200, frame)
            if frame != rr.WORLD:
                pnt[:, :2] *= 0.5
            x, geom, nrm = e.cast(q, pnt, vec, frame=frame, fb=fb)
            wp, wv = scene.to_world(frame, fb, pnt.astype(np.float32), vec.astype(np.float32))
            amb, dist_ok, nerr = compare(m, scene, wp, wv, x, geom, nrm, rb)
            assert dist_ok, frame
            assert nerr < 2e-3, (frame, nerr)
            n_amb += amb
            n_all += len(x)
            n_hit += int((geom >= 0).sum())
    body.close()
    e.close()
    assert n_hit > 0.3 * n_all, (n_hit, n_all)
    assert n_amb <= 0.03 * n_all, (task, n_amb, n_all)


# ---------------------------------------------------------------------------------------------------------------------
# header, Python layer, camera
# ---------------------------------------------------------------------------------------------------------------------
def test_header_constants_match_the_package(tmp_path):
    from loco_mujoco_b200 import engine
    src = tmp_path / "ray.c"
    src.write_text('#include <stdio.h>\n#include "locosim.h"\nint main(void) {\n'
                   '  printf("%d %d %d %d %d %d %d\\n", LS_RAY_WORLD, LS_RAY_BODY, LS_RAY_HEADING, LS_RAY_TRACK,'
                   " LS_RAY_STATIC, LS_RAY_DYNAMIC, LS_RAY_PER_ENV);\n  return 0; }\n")
    exe = tmp_path / "ray"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    v = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert v == [engine.RAY_WORLD, engine.RAY_BODY, engine.RAY_HEADING, engine.RAY_TRACK, engine.RAY_STATIC,
                 engine.RAY_DYNAMIC, engine.RAY_PER_ENV]


def _fake_engine(monkeypatch, calls):
    import torch
    from loco_mujoco_b200 import engine as engine_mod
    eng = object.__new__(engine_mod.CudaEngine)
    eng.torch = torch
    eng.n_envs, eng.nbody, eng.device, eng.h, eng.launches = 4, 5, torch.device("cpu"), None, 0
    eng.lib = types.SimpleNamespace(locosim_ray=lambda *a: calls.append(a) or 0)
    monkeypatch.setattr(engine_mod, "_ptr", lambda t: None if t is None else t.data_ptr())
    monkeypatch.setattr(engine_mod.CudaEngine, "_stream", lambda self: None)
    return eng


def test_ray_validates_its_arguments(monkeypatch):
    """null buffers, n_rays < 1, unknown frames and flag bits, bodies out of range, dtypes, shapes, devices and overlaps are
    refused before the engine is called"""
    import torch
    from loco_mujoco_b200 import engine as E
    calls = []
    eng = _fake_engine(monkeypatch, calls)
    pnt, vec = torch.zeros((7, 3)), torch.zeros((7, 3))
    dist, geom, nrm = torch.zeros((4, 7)), torch.zeros((4, 7), dtype=torch.int32), torch.zeros((4, 7, 3))
    eng.ray(pnt, vec, dist, geom, nrm, frame=E.RAY_BODY, frame_body=4, exclude_body=-1)
    eng.ray(torch.zeros((4, 7, 3)), torch.zeros((4, 7, 3)), dist, geom, flags=E.RAY_STATIC | E.RAY_PER_ENV)
    eng.ray(pnt, pnt, dist, geom)                                            # the inputs may share memory
    assert len(calls) == 3 and calls[0][3:8] == (7, E.RAY_BODY, 4, -1, E.RAY_STATIC | E.RAY_DYNAMIC)
    big = torch.zeros(4 * 7 * 5)
    bad = [dict(pnt=None), dict(vec=None), dict(dist=None), dict(geom=None),
           dict(pnt=torch.zeros((0, 3)), vec=torch.zeros((0, 3)), dist=torch.zeros((4, 0)),
                geom=torch.zeros((4, 0), dtype=torch.int32), normal=None),          # n_rays < 1
           dict(frame=4), dict(frame=-1), dict(flags=8), dict(frame_body=5), dict(frame_body=-1),
           dict(exclude_body=5), dict(exclude_body=-2),
           dict(pnt=pnt.double()), dict(geom=geom.float()), dict(dist=dist.int()), dict(vec=torch.zeros((7, 4))),
           dict(dist=torch.zeros((4, 8))), dict(normal=torch.zeros((4, 7, 2))), dict(pnt=torch.zeros((3, 7)).t()),
           dict(flags=E.RAY_PER_ENV | E.RAY_STATIC),                                 # per-env rays need [n, r, 3]
           dict(dist=big[:28].view(4, 7), normal=big[20:104].view(4, 7, 3)),         # outputs overlap
           dict(pnt=big[:21].view(7, 3), dist=big[:28].view(4, 7)),                  # an output overlaps an input
           dict(vec=nrm.view(-1)[:21].view(7, 3))]
    for b in bad:
        kw = dict(pnt=pnt, vec=vec, dist=dist, geom=geom, normal=nrm)
        kw.update(b)
        args = {k: kw.pop(k) for k in ("pnt", "vec", "dist", "geom", "normal")}
        with pytest.raises(ValueError):
            eng.ray(args["pnt"], args["vec"], args["dist"], args["geom"], args["normal"], **kw)
    assert len(calls) == 3
    eng.device = torch.device("cuda", 0)                                                 # another device
    with pytest.raises(ValueError):
        eng.ray(pnt, vec, dist, geom)
    assert len(calls) == 3


class _CameraEngine:
    """Stands in for CudaEngine on a CPU-only box: every ray hits geom 0 at dist 2 (units of |vec|), and records what was
    asked"""

    def __init__(self, model_blobs, task_blobs, n_envs, device=0, **kw):
        import torch
        self.device, self.n_envs, self.calls = torch.device("cpu"), n_envs, []

    def ray(self, pnt, vec, dist, geom, normal=None, frame=0, frame_body=0, exclude_body=-1, flags=3):
        self.calls.append((pnt, vec, frame, frame_body, exclude_body, flags))
        dist.fill_(2.0)
        geom.fill_(0)
        if normal is not None:
            normal.zero_()
        return dist, geom, normal

    def set_param_pool(self, pool):
        pass

    def close(self):
        pass


def test_camera_ray_geometry(bundled_only, monkeypatch):
    """the centre of the image is on the optical axis, the top and bottom image edges are at +-fovy / 2, rows run top to
    bottom and columns left to right, vec has unit length, and depth = dist (dir . axis)"""
    import torch
    from loco_mujoco_b200 import engine as engine_mod
    monkeypatch.setattr(engine_mod, "CudaEngine", _CameraEngine)
    env = _make("UnitreeA1.simple", num_envs=3)
    W, H, fovy, az, el = 8, 6, 60.0, 30.0, -25.0
    cam = env.camera(W, H, fovy=fovy, azimuth=az, elevation=el, distance=2.0)
    eng = env._get_engine()
    pnt, vec, frame, fb, ex, flags = eng.calls[-1]
    assert frame == engine_mod.RAY_TRACK and fb == 1 and ex == -1 and flags == engine_mod.RAY_STATIC | engine_mod.RAY_DYNAMIC
    a, e = np.radians(az), np.radians(el)
    axis = np.array([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)])
    up = np.array([-np.sin(e) * np.cos(a), -np.sin(e) * np.sin(a), np.cos(e)])
    right = np.cross(axis, up)
    assert np.allclose(pnt.numpy(), -2.0 * axis, atol=1e-6)
    d = vec.numpy().reshape(H, W, 3).astype(np.float64)
    assert np.allclose(np.linalg.norm(d, axis=-1), 1, atol=1e-6)
    centre = d[H // 2 - 1:H // 2 + 1, W // 2 - 1:W // 2 + 1].sum((0, 1))
    assert np.allclose(centre / np.linalg.norm(centre), axis, atol=1e-6)
    # vertical angle of row i's centre: tan = (H/2 - i - 0.5) / (H/2) tan(fovy/2), so the image edges are at +-fovy/2
    t = np.tan(np.radians(fovy) / 2)
    for i in range(H):
        for j in (0, W - 1):
            r = d[i, j]
            assert abs((r @ up) / (r @ axis) - (H / 2 - i - 0.5) / (H / 2) * t) < 1e-6
            assert abs((r @ right) / (r @ axis) - (j + 0.5 - W / 2) / (H / 2) * t) < 1e-6
    assert np.allclose(cam["depth"].numpy(), 2.0 * (d @ axis)[None], atol=1e-6)
    assert tuple(cam["geom"].shape) == (3, H, W) and tuple(cam["body"].shape) == (3, H, W)
    assert int(cam["body"].max()) == int(env._model.geom_bodyid[0])
    # "body" mode: the camera looks along its frame's -z with y up, in the body's frame
    cam2 = env.camera(4, 4, mode="body", body="trunk", pos=(0.1, 0, 0.05), quat=(1, 0, 0, 0), out=None)
    pnt, vec, frame, fb, _, _ = eng.calls[-1]
    assert frame == engine_mod.RAY_BODY and fb == env.body_index("trunk")
    assert np.allclose(pnt.numpy()[0], [0.1, 0, 0.05]) and (vec.numpy()[:, 2] < 0).all()
    # refilled in place
    again = env.camera(4, 4, mode="body", body="trunk", pos=(0.1, 0, 0.05), quat=(1, 0, 0, 0), out=cam2)
    assert again is cam2 and again["_rays"]["dist"] is cam2["_rays"]["dist"]


def test_ray_cast_arguments(bundled_only, monkeypatch):
    import torch
    from loco_mujoco_b200 import engine as engine_mod
    monkeypatch.setattr(engine_mod, "CudaEngine", _CameraEngine)
    env = _make("UnitreeA1.simple", num_envs=3)
    eng = env._get_engine()
    r = env.ray_cast(torch.zeros((5, 3)), torch.ones((5, 3)), frame="trunk", mode="heading", exclude_body="trunk",
                     static=False, normal=True)
    _, _, frame, fb, ex, flags = eng.calls[-1]
    assert (frame, fb, ex, flags) == (engine_mod.RAY_HEADING, env.body_index("trunk"), env.body_index("trunk"),
                                      engine_mod.RAY_DYNAMIC)
    assert set(r) == {"dist", "geom", "normal"} and tuple(r["normal"].shape) == (3, 5, 3)
    r2 = env.ray_cast(torch.zeros((3, 5, 3)), torch.ones((3, 5, 3)), out=r)
    assert r2 is r and eng.calls[-1][2:] == (engine_mod.RAY_WORLD, 0, -1, 7)
    for bad in (dict(mode="camera"), dict(frame="no such body", mode="body"), dict(frame=99, mode="body"),
                dict(exclude_body=-3), dict(out=[1])):
        with pytest.raises(ValueError):
            env.ray_cast(torch.zeros((5, 3)), torch.ones((5, 3)), **bad)


def test_4ages_all_refuses_ray_casting(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    env = LocoEnv.make("HumanoidTorque4Ages.walk.all.real", num_envs=8, debug=True)
    for f in (lambda: env.ray_cast(None, None), lambda: env.camera(4, 4), lambda: env.render()):
        with pytest.raises(NotImplementedError):
            f()
