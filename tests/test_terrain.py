"""Height-field terrain (include/locosim.h locosim_set_terrain_origin) without a GPU: the ModelPack stays byte for byte what it
was for every model without a terrain; the fp64 reference (tests/csrc/terrain_ref.c) against closed-form geometry; the serial
build of the engine's terrain configuration against that reference (contact lists in order, rollouts of UnitreeA1); and
the Python side (loco_mujoco_b200/terrain.py, LocoEnv's terrain=)."""
import ctypes
import glob
import hashlib
import os

import numpy as np
import pytest

import terrain_ref
from helpers import ROOT, make_env

GEOM_SPHERE, GEOM_CAPSULE, GEOM_CYLINDER, GEOM_BOX = 2, 3, 5, 6
# MPR stops when its portal is within opt.mpr_tolerance = 1e-6 of the Minkowski difference's surface: normals and depths of
# curved geoms are exact to that tolerance, not to round-off
MPR_TOL = 1e-6

PARENT_PACK_SHA256 = {
    "Atlas.carry.npz|model0|0": "2d9b63b7d88b57e6",
    "Atlas.carry.npz|model0|1": "2d9b63b7d88b57e6",
    "Atlas.carry.npz|model1|0": "4a3f739b4fdff089",
    "Atlas.carry.npz|model1|1": "4a3f739b4fdff089",
    "Atlas.carry.npz|model2|0": "c1b2caf306784e18",
    "Atlas.carry.npz|model2|1": "c1b2caf306784e18",
    "Atlas.carry.npz|model3|0": "c06ff0e93d854151",
    "Atlas.carry.npz|model3|1": "c06ff0e93d854151",
    "Atlas.walk.npz|model|0": "89ec37a1a0ab71fd",
    "Atlas.walk.npz|model|1": "89ec37a1a0ab71fd",
    "HumanoidTorque.run.npz|model|0": "53eb87ea339dc248",
    "HumanoidTorque.run.npz|model|1": "cffc6fda51125a59",
    "HumanoidTorque.walk.npz|model|0": "53eb87ea339dc248",
    "HumanoidTorque.walk.npz|model|1": "cffc6fda51125a59",
    "HumanoidTorque4Ages.run.1.npz|model|0": "8dc338b73f375ceb",
    "HumanoidTorque4Ages.run.1.npz|model|1": "1a4748d60fcbb795",
    "HumanoidTorque4Ages.run.2.npz|model|0": "b1680638f51e139e",
    "HumanoidTorque4Ages.run.2.npz|model|1": "6519e835851faf99",
    "HumanoidTorque4Ages.run.3.npz|model|0": "c1bd13dd70d25156",
    "HumanoidTorque4Ages.run.3.npz|model|1": "cf9ec482857eb4bd",
    "HumanoidTorque4Ages.run.4.npz|model|0": "53eb87ea339dc248",
    "HumanoidTorque4Ages.run.4.npz|model|1": "cffc6fda51125a59",
    "HumanoidTorque4Ages.walk.1.npz|model|0": "8dc338b73f375ceb",
    "HumanoidTorque4Ages.walk.1.npz|model|1": "1a4748d60fcbb795",
    "HumanoidTorque4Ages.walk.2.npz|model|0": "b1680638f51e139e",
    "HumanoidTorque4Ages.walk.2.npz|model|1": "6519e835851faf99",
    "HumanoidTorque4Ages.walk.3.npz|model|0": "c1bd13dd70d25156",
    "HumanoidTorque4Ages.walk.3.npz|model|1": "cf9ec482857eb4bd",
    "HumanoidTorque4Ages.walk.4.npz|model|0": "53eb87ea339dc248",
    "HumanoidTorque4Ages.walk.4.npz|model|1": "cffc6fda51125a59",
    "Talos.carry.npz|model0|0": "ae60ed5487d998b3",
    "Talos.carry.npz|model0|1": "ae60ed5487d998b3",
    "Talos.carry.npz|model1|0": "8b8501195dc29e17",
    "Talos.carry.npz|model1|1": "8b8501195dc29e17",
    "Talos.carry.npz|model2|0": "90f4b8ba6831fd61",
    "Talos.carry.npz|model2|1": "90f4b8ba6831fd61",
    "Talos.carry.npz|model3|0": "fb68ee3001c4967c",
    "Talos.carry.npz|model3|1": "fb68ee3001c4967c",
    "Talos.walk.npz|model|0": "91b6044c5aa96c27",
    "Talos.walk.npz|model|1": "91b6044c5aa96c27",
    "UnitreeA1.hard.npz|model|0": "2fceb2b5ce1a80a2",
    "UnitreeA1.hard.npz|model|1": "c5c86322149154e2",
    "UnitreeA1.simple.npz|model|0": "2fceb2b5ce1a80a2",
    "UnitreeA1.simple.npz|model|1": "c5c86322149154e2",
    "UnitreeG1.run.npz|model|0": "d7f28421a302f34a",
    "UnitreeG1.run.npz|model|1": "12cddfa27621530a",
    "UnitreeG1.walk.npz|model|0": "d7f28421a302f34a",
    "UnitreeG1.walk.npz|model|1": "12cddfa27621530a",
    "UnitreeH1.carry.npz|model0|0": "3bb2d3a90bc624dd",
    "UnitreeH1.carry.npz|model0|1": "1436b1baa5d2966a",
    "UnitreeH1.carry.npz|model1|0": "28f37f240cbc0bc3",
    "UnitreeH1.carry.npz|model1|1": "cb2f60d89000c10d",
    "UnitreeH1.carry.npz|model2|0": "aa21047be9dda7cf",
    "UnitreeH1.carry.npz|model2|1": "7ba1bc0574cce32f",
    "UnitreeH1.carry.npz|model3|0": "636c40a780d9f721",
    "UnitreeH1.carry.npz|model3|1": "c85dbce41947fabd",
    "UnitreeH1.run.npz|model|0": "45072923ad5ec001",
    "UnitreeH1.run.npz|model|1": "467e2d783352d16a",
    "UnitreeH1.walk.npz|model|0": "45072923ad5ec001",
    "UnitreeH1.walk.npz|model|1": "467e2d783352d16a",
}


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def ref():
    return terrain_ref.load()


@pytest.fixture(scope="module")
def emu_t(emu):
    emu.emu_set_terrain_origin.restype = None
    emu.emu_set_terrain_origin.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    emu.emu_select_cfg.restype = ctypes.c_int
    emu.emu_select_cfg.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    emu.emu_ncon.restype = ctypes.c_int
    emu.emu_ncon.argtypes = [ctypes.c_void_p]
    emu.emu_contact.restype = None
    emu.emu_contact.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    emu.emu_max_contacts.restype = ctypes.c_int
    emu.emu_max_contacts.argtypes = [ctypes.c_void_p]
    emu.emu_forward.restype = None
    emu.emu_forward.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    return emu


# ---------------------------------------------------------------------------------------------------------------------
# 1. nothing existing changed
# ---------------------------------------------------------------------------------------------------------------------
def test_bundled_assets_pack_to_the_parent_bytes():
    """Every bundled model, with and without its convex pairs, packs to the same bytes as before the terrain existed
    (SHA-256 prefixes recorded from the parent's modelpack.pack): LOCOSIM_MP_VERSION is kept."""
    from loco_mujoco_b200 import modelpack
    seen = 0
    for f in sorted(glob.glob(os.path.join(ROOT, "loco_mujoco_b200", "assets", "*.npz"))):
        a = np.load(f, allow_pickle=False)
        for pre in sorted(set(k.split("_")[0] for k in a.files if k.startswith("model"))):
            m = modelpack.from_npz_dict({k[len(pre) + 1:]: a[k] for k in a.files if k.startswith(pre + "_")})
            for cp in (True, False):
                ints, reals = modelpack.pack(m, convex_pairs=cp)
                key = "%s|%s|%d" % (os.path.basename(f), pre, cp)
                assert hashlib.sha256(ints.tobytes() + reals.tobytes()).hexdigest()[:16] == PARENT_PACK_SHA256[key], key
                assert not ints[11:13].any() and not reals[7:11].any()
                seen += 1
    assert seen == len(PARENT_PACK_SHA256)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the fp64 reference against geometry
# ---------------------------------------------------------------------------------------------------------------------
def _rot(axis, ang):
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _lowest(gtype, mat, size):
    """half extent of the geom along z (its lowest point lies that far below its centre)"""
    a = abs(mat[2, 2])
    if gtype == GEOM_SPHERE:
        return size[0]
    if gtype == GEOM_CAPSULE:
        return size[0] + size[1] * a
    if gtype == GEOM_CYLINDER:
        return size[0] * np.sqrt(max(1 - a * a, 0)) + size[1] * a
    return np.abs(mat[2]) @ size


FLAT = np.zeros((9, 9))
SIZE4 = np.array([1.0, 1.0, 0.0, 0.5])


@pytest.mark.parametrize("gtype,size,mat", [
    (GEOM_SPHERE, [0.02, 0, 0], np.eye(3)),
    (GEOM_CAPSULE, [0.03, 0.1, 0], _rot([1, 0.3, 0], 1.2)),
    (GEOM_CYLINDER, [0.04, 0.06, 0], _rot([0.2, 1, 0], 0.4)),
    (GEOM_BOX, [0.05, 0.03, 0.02], _rot([1, 1, 1], 0.7)),
])
def test_flat_field_gives_up_normals_and_the_depth(ref, gtype, size, mat):
    size = np.asarray(size, float)
    h = 0.25
    pen = 0.004
    pos = np.array([0.13, -0.21, h + _lowest(gtype, mat, size) - pen])
    con, _ = terrain_ref.debug_geom(ref, FLAT, [1.0, 1.0, 0.0, 0.5], [0, 0, h], [0, 0], gtype, pos, mat, size)
    # one contact per penetrated prism: the deepest has the field's normal and the geom's depth; a prism the geom only
    # grazes near its side gives a shallower contact (MPR's least-depth direction through that side)
    assert len(con) >= 1
    k = int(np.argmin(con[:, 0]))
    np.testing.assert_allclose(con[k, 4:7], [0, 0, 1.0], atol=2 * MPR_TOL)
    np.testing.assert_allclose(con[k, 0], -pen, atol=MPR_TOL)
    assert np.all(con[:, 0] >= -pen - MPR_TOL)


def test_planar_slope_gives_its_normal_and_the_analytic_depth(ref):
    nrow, ncol, rx, ry = 11, 13, 1.0, 1.2
    x = np.linspace(-rx, rx, ncol)
    y = np.linspace(-ry, ry, nrow)
    a, b, c0 = 0.2, -0.15, 0.5
    Z = c0 + a * x[None, :] + b * y[:, None]
    from loco_mujoco_b200.terrain import HeightField
    hf = HeightField(Z, (rx, ry), base=0.5)
    n = np.array([-a, -b, 1.0]) / np.sqrt(1 + a * a + b * b)
    r = 0.05
    p = np.array([0.1, 0.2, 0.0])
    surf = c0 + a * p[0] + b * p[1]
    pen = 0.01
    p[2] = surf + (r - pen) / n[2]                     # centre r - pen from the plane along its normal
    con, _ = terrain_ref.debug_geom(ref, hf.data, hf.size4, hf.geom_pos, [0, 0], GEOM_SPHERE, p, np.eye(3), [r, 0, 0])
    assert len(con) >= 1
    k = int(np.argmin(con[:, 0]))
    np.testing.assert_allclose(con[k, 4:7], n, atol=2 * MPR_TOL)
    np.testing.assert_allclose(con[k, 0], -pen, atol=MPR_TOL)
    assert np.all(con[:, 0] >= -pen - MPR_TOL)


def test_sphere_in_a_v_valley_gets_one_contact_per_face(ref):
    ncol, nrow = 3, 2
    s = 0.5
    Z = np.array([[s, 0.0, s], [s, 0.0, s]])            # valley along y at x = 0, faces slope 0.5 in x
    size4 = [1.0, 1.0, s, 0.5]
    r = 0.2
    zc = r / np.cos(np.arctan(s)) - 0.01                # touching both faces, 1 cm too low
    con, _ = terrain_ref.debug_geom(ref, Z / s, size4, [0, 0, 0], [0, 0], GEOM_SPHERE, [0, 0, zc], np.eye(3), [r, 0, 0])
    nl = np.array([s, 0, 1]) / np.sqrt(1 + s * s)       # the left face (x < 0) rises to the left: normal leans +x
    nr = np.array([-s, 0, 1]) / np.sqrt(1 + s * s)
    normals = con[:, 4:7]
    assert len(con) >= 2
    assert all(np.allclose(n, nl, atol=MPR_TOL) or np.allclose(n, nr, atol=MPR_TOL) for n in normals)
    assert any(np.allclose(n, nl, atol=MPR_TOL) for n in normals) and any(np.allclose(n, nr, atol=MPR_TOL) for n in normals)


def test_geom_outside_the_field_box_gets_none(ref):
    for p in ([1.5, 0, 0], [0, -1.5, 0], [0, 0, 0.9], [0, 0, -0.9]):
        con, nm = terrain_ref.debug_geom(ref, FLAT, SIZE4, [0, 0, 0], [0, 0], GEOM_SPHERE, p, np.eye(3), [0.1, 0, 0])
        assert len(con) == 0 and nm == 0


def test_sphere_straddling_a_cell_boundary_gets_one_contact_per_penetrated_prism(ref):
    dx = 2.0 / 8
    p = np.array([-1 + 3 * dx, -1 + 4 * dx + 0.003, 0.018])   # on the vertical grid line x = 3 dx, near row 4's edge
    con, nm = terrain_ref.debug_geom(ref, FLAT, SIZE4, [0, 0, 0], [0, 0], GEOM_SPHERE, p, np.eye(3), [0.02, 0, 0])
    # the prisms whose top triangle reaches into the disc |xy - p| < sqrt(r^2 - z^2) all penetrate
    assert len(con) >= 2 and len(con) <= nm
    # (MPR's depth near a prism's edge is good to its portal, ~1e-4 here)
    assert np.all(con[:, 0] >= -0.002 - 1e-4) and abs(np.median(con[:, 0]) + 0.002) < 2e-4


def test_origin_shift_equals_moving_the_geom(ref):
    rng = np.random.RandomState(3)
    Z = rng.uniform(0, 1, (17, 19))
    size4 = [2.0, 1.5, 0.3, 0.5]
    p = np.array([0.3, -0.2, 0.12])
    d = np.array([0.77, -0.41])
    mat = _rot([0.3, 1, 0.2], 0.9)
    a, _ = terrain_ref.debug_geom(ref, Z, size4, [0, 0, 0], d, GEOM_CAPSULE, p, mat, [0.03, 0.08, 0])
    b, _ = terrain_ref.debug_geom(ref, Z, size4, [0, 0, 0], [0, 0], GEOM_CAPSULE, p + np.r_[d, 0], mat, [0.03, 0.08, 0])
    assert len(a) == len(b) and len(a) > 0
    np.testing.assert_allclose(a[:, 0], b[:, 0], atol=1e-12)
    np.testing.assert_allclose(a[:, 4:7], b[:, 4:7], atol=1e-12)
    np.testing.assert_allclose(a[:, 1:4] + np.r_[d, 0], b[:, 1:4], atol=1e-12)


def test_fifty_contacts_per_pair_at_most(ref):
    Z = np.zeros((41, 41))
    con, nm = terrain_ref.debug_geom(ref, Z, [1.0, 1.0, 0.0, 0.5], [0, 0, 0], [0, 0], GEOM_BOX, [0, 0, 0.09], np.eye(3),
                                     [0.4, 0.4, 0.1])
    assert len(con) == terrain_ref.MAXCONPAIR and nm >= terrain_ref.MAXCONPAIR


# ---------------------------------------------------------------------------------------------------------------------
# 3. the serial build of the engine's terrain configuration against the reference
# ---------------------------------------------------------------------------------------------------------------------
def _a1_on(hf, **kw):
    return make_env("UnitreeA1.simple", terrain=hf, **kw)


def _rough(seed=1, res=0.05):
    from loco_mujoco_b200 import terrain
    return terrain.tiled_terrain(n_rows=2, n_cols=4, tile_size=2.0, resolution=res, max_rough=0.04, max_slope=0.25,
                                 max_step=0.06, step_width=0.2, platform=0.4, base=0.1, seed=seed)


def _start(env):
    from helpers import golden
    spec = env.task_spec()
    g = golden("UnitreeA1.simple")
    q, v = np.zeros(env._model.nq), np.zeros(env._model.nq)
    for t, i, val in zip(spec.obs_src_type, spec.obs_src_idx, g[0]):
        if t == 0:
            q[i] = val
        elif t == 1:
            v[i] = val
    return q, v


def test_terrain_model_selects_the_terrain_configuration(emu_t, bundled_only):
    from loco_mujoco_b200 import modelpack
    env = _a1_on(_rough())
    ints, reals = modelpack.pack(env._model)
    assert emu_t.emu_select_cfg(_p(ints), len(ints), _p(reals), len(reals)) == 6
    assert env.geom_names[-1] == "terrain" and env.geom_index("terrain") == env._model.ngeom - 1
    assert env._model.ngeom == 39
    m0 = make_env("UnitreeA1.simple")._model
    i0, r0 = modelpack.pack(m0)
    assert emu_t.emu_select_cfg(_p(i0), len(i0), _p(r0), len(r0)) == 0


@pytest.mark.parametrize("origin", [(0.0, 0.0), (1.0, -1.0), (-3.0, 1.0)])
def test_serial_engine_matches_the_reference_on_rough_terrain(emu_t, ref, bundled_only, origin):
    """UnitreeA1 under seeded random actions on a tiled rough field: the contact list of every step's last evaluation in
    order, and the state, against the fp64 reference (the tolerance of the serial-versus-oracle rollout tests)."""
    from loco_mujoco_b200 import modelpack
    env = _a1_on(_rough())
    spec = env.task_spec()
    ints, reals = modelpack.pack(env._model)
    sim = emu_t.emu_create(_p(ints), len(ints), _p(reals), len(reals))
    o32 = np.array(origin, dtype=np.float32)
    emu_t.emu_set_terrain_origin(sim, _p(o32))
    rs = terrain_ref.Sim(ref, (ints, reals))
    rs.set_origin(o32.astype(np.float64))
    q, v = _start(env)
    emu_t.emu_reset(sim, _p(q), _p(v))
    rs.reset(q, v)
    rng = np.random.RandomState(7)
    qe, ve = np.zeros(len(q)), np.zeros(len(q))
    worst, n_terr = 0.0, 0
    for k in range(30):
        a = rng.uniform(-1, 1, env._model.nu) * 0.3
        ctrl = np.zeros(env._model.nu)
        ctrl[spec.act_idx] = a * spec.act_delta + spec.act_mean
        # contact lists of the same state
        emu_t.emu_forward(sim, _p(ctrl))
        rs.forward(ctrl)
        ce = []
        for c in range(emu_t.emu_ncon(sim)):
            o = np.zeros(18)
            emu_t.emu_contact(sim, c, _p(o))
            ce.append(o)
        # (the engine keeps the contacts inside the pair's inclusion distance only: margin - gap)
        mg, gp = np.asarray(env._model.geom_margin), np.asarray(env._model.geom_gap)
        cr = [r for r in rs.contacts() if r[0] < max(mg[int(r[7])], mg[int(r[8])]) - max(gp[int(r[7])], gp[int(r[8])])]
        cap = emu_t.emu_max_contacts(sim)
        # the engine's list is the reference's, up to the per-env caps of the contact list (16) and of the contact rows
        # (64: make_constraint drops the tail that does not fit, DESIGN.md section 7); where neither binds, all of it
        rows = np.cumsum([int(r[9]) for r in cr])
        n_fit = min(cap, int(np.searchsorted(rows, 64, side="right")))
        if n_fit == len(cr):
            assert len(ce) == len(cr), (k, len(ce), len(cr))
        assert len(ce) <= n_fit
        assert [(int(o[0]), int(o[1])) for o in ce] == [(int(r[7]), int(r[8])) for r in cr[:len(ce)]], k
        for o, r in zip(ce, cr):
            assert abs(o[3] - r[0]) < 5e-4, k          # (fp32 MPR on tall, thin prisms: DESIGN.md section 6)
            # the normal of a contact through a prism's top: a geom grazing a prism's side can end fp32 MPR on another
            # final portal than fp64, with another normal and point for the same depth (DESIGN.md section 7)
            if r[6] > 0.99 and o[14] > 0.99:
                np.testing.assert_allclose(o[12:15], r[4:7], atol=6e-2)      # (measured: 3.9e-2)
        n_terr += sum(int(o[0]) == env._model.ngeom - 1 for o in ce)
        emu_t.emu_reset(sim, _p(q), _p(v))          # (forward moved nothing; restart the step from the same state)
        emu_t.emu_step(sim, _p(ctrl), spec.n_substeps)
        rs.step(ctrl, spec.n_substeps)
        emu_t.emu_get_state(sim, _p(qe), _p(ve))
        q, v = rs.state()
        worst = max(worst, float(np.abs(qe - q).max()))
        emu_t.emu_reset(sim, _p(q), _p(v))
    emu_t.emu_destroy(sim)
    rs.close()
    assert n_terr > 0
    # (one control step from the same state: measured up to 6.2e-3 on this field, against 2e-3 of the plane-only models;
    # the wider bound is DESIGN.md section 6's, its cause section 7's)
    assert worst < 1e-2, worst


# ---------------------------------------------------------------------------------------------------------------------
# 5. statics: A1 at rest on a raised flat field carries its weight through the terrain alone (tests/test_foot_forces.py
#    checks the same on the plane)
# ---------------------------------------------------------------------------------------------------------------------
def test_a1_at_rest_on_a_raised_field_carries_its_weight(ref, bundled_only):
    from loco_mujoco_b200 import modelpack
    from loco_mujoco_b200.terrain import HeightField
    lift = 0.3
    env = _a1_on(HeightField(np.full((41, 41), lift), (2.0, 2.0), base=0.5))
    m, spec = env._model, env.task_spec()
    rs = terrain_ref.Sim(ref, modelpack.pack(m))
    q, v = _start(env)
    q[m.joint_id("trunk_tz")] += lift
    rs.reset(q, v)
    ctrl = np.zeros(m.nu)
    ctrl[spec.act_idx] = spec.act_mean                        # zero action: the robot collapses and comes to rest
    for _ in range(250):
        rs.step(ctrl, spec.n_substeps)
    q, v = rs.state()
    assert np.abs(v).max() < 5e-2, "not at rest"
    rs.forward(ctrl)
    con = rs.contacts()
    assert len(con) > 0 and np.all(con[:, 7] == m.ngeom - 1), "the floor is 0.3 m below: only the terrain carries the robot"
    # (a foot that reaches over a prism's edge also gets a contact through the prism's side: sum the world z force of each
    # contact, its frame rebuilt from the normal as mju_makeFrame builds it)
    total = 0.0
    for r in con:
        n = r[4:7]
        t1 = np.array([0, 1.0, 0]) if abs(n[1]) < 0.5 else np.array([0, 0, 1.0])
        t1 = t1 - n.dot(t1) * n
        t1 /= np.linalg.norm(t1)
        t2 = np.cross(n, t1)
        total += r[10] * n[2] + r[11] * t1[2] + r[12] * t2[2]
    weight = float(np.sum(m.body_mass)) * 9.81
    assert abs(total - weight) < 0.01 * weight, (total, weight)
    rs.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. Python
# ---------------------------------------------------------------------------------------------------------------------
def test_heightfield_round_trips_metres():
    from loco_mujoco_b200.terrain import HeightField
    rng = np.random.RandomState(0)
    H = rng.uniform(-0.3, 0.7, (5, 7))
    hf = HeightField(H, (1.0, 2.0), base=0.2, pos=(0.5, -0.5, 0.1))
    np.testing.assert_allclose(hf.heights(), H + 0.1, atol=1e-12)
    assert hf.data.min() == 0.0 and hf.data.max() == 1.0
    np.testing.assert_allclose(hf.size4, [1.0, 2.0, 1.0 * (H.max() - H.min()), 0.2])
    assert hf.geom_pos[2] == pytest.approx(0.1 + H.min())
    x, y = hf.sample_xy()
    np.testing.assert_allclose(x, np.linspace(-0.5, 1.5, 7))
    np.testing.assert_allclose(y, np.linspace(-2.5, 1.5, 5))
    flat = HeightField(np.full((2, 2), 0.4), (1, 1))
    assert flat.elevation == 0 and np.all(flat.heights() == 0.4)


@pytest.mark.parametrize("kw,msg", [
    (dict(heights_m=np.zeros(4), size=(1, 1)), "nrow, ncol >= 2"),
    (dict(heights_m=np.zeros((1, 4)), size=(1, 1)), "nrow, ncol >= 2"),
    (dict(heights_m=np.full((2, 2), np.nan), size=(1, 1)), "finite"),
    (dict(heights_m=np.zeros((2, 2)), size=(0, 1)), "rx, ry > 0"),
    (dict(heights_m=np.zeros((2, 2)), size=(1, 1, 1)), "rx, ry > 0"),
    (dict(heights_m=np.zeros((2, 2)), size=(1, 1), base=0), "base must be positive"),
    (dict(heights_m=np.zeros((2, 2)), size=(1, 1), pos=(0, 0)), "pos must be"),
])
def test_heightfield_argument_checks(kw, msg):
    from loco_mujoco_b200.terrain import HeightField
    with pytest.raises(ValueError, match=msg):
        HeightField(**kw)


def test_generator_is_deterministic_and_its_platforms_are_at_zero():
    from loco_mujoco_b200 import terrain
    a, b, c = (terrain.tiled_terrain(n_rows=3, n_cols=4, tile_size=4.0, resolution=0.1, seed=s) for s in (5, 5, 6))
    assert np.array_equal(a.heights(), b.heights()) and not np.array_equal(a.heights(), c.heights())
    o = a.tile_origins()
    assert o.shape == (12, 2)
    x, y = a.sample_xy()
    H = a.heights()
    for ox, oy in o:
        near = (np.abs(x[None, :] - ox) <= 0.5 + 1e-9) & (np.abs(y[:, None] - oy) <= 0.5 + 1e-9)
        assert near.sum() == 121 and np.abs(H[near]).max() < 1e-12
    # difficulty grows with the row: the stairs column gets deeper
    assert H.min() < -0.05
    with pytest.raises(ValueError, match="even integer"):
        terrain.tiled_terrain(tile_size=1.0, resolution=0.3)
    with pytest.raises(ValueError, match="unknown tile kind"):
        terrain.tiled_terrain(kinds=("lava",))
    with pytest.raises(ValueError, match="not a tiled_terrain"):
        terrain.HeightField(np.zeros((2, 2)), (1, 1)).tile_origins()


def test_terrain_on_another_robot_is_refused(bundled_only):
    from loco_mujoco_b200.terrain import HeightField
    with pytest.raises(NotImplementedError, match="UnitreeA1 only"):
        make_env("Atlas.walk", terrain=HeightField(np.zeros((2, 2)), (1, 1)))
    with pytest.raises(NotImplementedError, match="domain_randomization_config"):
        make_env("UnitreeA1.simple", terrain=HeightField(np.zeros((2, 2)), (1, 1)), domain_randomization_config="dr.yaml")
    with pytest.raises(TypeError, match="HeightField"):
        make_env("UnitreeA1.simple", terrain=np.zeros((2, 2)))


def test_terrain_pairs_copy_the_floor(bundled_only):
    from loco_mujoco_b200 import modelpack
    env = _a1_on(_rough())
    m = env._model
    t = m.ngeom - 1
    pg = np.asarray(m.pair_geom).reshape(-1, 2)
    floor = [g for g in range(t) if m.geom_type[g] == 0][0]
    assert sorted(pg[pg[:, 0] == t, 1]) == sorted(pg[pg[:, 0] == floor, 1])
    for f in ("geom_friction", "geom_solref", "geom_solimp", "geom_margin", "geom_gap", "geom_condim", "geom_priority",
              "geom_solmix", "geom_contype", "geom_conaffinity"):
        a = np.asarray(getattr(m, f))
        np.testing.assert_array_equal(a.reshape(m.ngeom, -1)[t], a.reshape(m.ngeom, -1)[floor])
    ints, reals = modelpack.pack(m)
    nrow, ncol = m.hfield.data.shape
    assert ints[11] == nrow and ints[12] == ncol
    np.testing.assert_array_equal(reals[-nrow * ncol:], m.hfield.data.ravel())
    assert env.terrain is m.hfield
    with pytest.raises(ValueError, match="no terrain"):
        make_env("UnitreeA1.simple").terrain_origin


# ---------------------------------------------------------------------------------------------------------------------
# 4. rays: the serial build's mj_rayHfield against the fp64 brute force (terrain_ref.ray_hfield)
# ---------------------------------------------------------------------------------------------------------------------
def _emu_rays(emu, env, origin, pnt, vec, flags=3, exclude=-1):
    from loco_mujoco_b200 import modelpack
    ints, reals = modelpack.pack(env._model)
    sim = emu.emu_create(_p(ints), len(ints), _p(reals), len(reals))
    o32 = np.array(origin, dtype=np.float32)
    emu.emu_set_terrain_origin(sim, _p(o32))
    q, v = _start(env)
    q[env._model.joint_id("trunk_tz")] += 5.0             # (the robot out of the way, above every ray)
    emu.emu_reset(sim, _p(q), _p(v))
    n = len(pnt)
    P, V = np.ascontiguousarray(pnt, np.float32), np.ascontiguousarray(vec, np.float32)
    d, g, nr = np.zeros(n, np.float32), np.zeros(n, np.int32), np.zeros((n, 3), np.float32)
    emu.emu_ray.restype = None
    emu.emu_ray.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int] * 5 + [ctypes.c_void_p] * 3
    emu.emu_ray(sim, _p(P), _p(V), n, 0, 0, exclude, flags, _p(d), _p(g), _p(nr))
    emu.emu_destroy(sim)
    return d, g, nr


def _stairs():
    from loco_mujoco_b200 import terrain
    return terrain.tiled_terrain(n_rows=1, n_cols=1, tile_size=4.0, resolution=0.05, kinds=("stairs",), max_step=0.1,
                                 step_width=0.3, platform=1.0, base=0.2, seed=0)


@pytest.mark.parametrize("origin", [(0.0, 0.0), (0.6, -0.35)])
def test_vertical_rays_return_the_height_of_the_triangle_under_them(emu_t, bundled_only, origin):
    hf = _rough(res=0.1)
    env = _a1_on(hf)
    rng = np.random.RandomState(2)
    xy = rng.uniform([-hf.rx, -hf.ry], [hf.rx, hf.ry], (200, 2)) - np.array(origin) + hf.geom_pos[:2]
    pnt = np.c_[xy, np.full(len(xy), 2.0)]
    vec = np.tile([0, 0, -1.0], (len(xy), 1))
    d, g, nr = _emu_rays(emu_t, env, origin, pnt, vec)
    tg = env._model.ngeom - 1
    for k in range(len(xy)):
        x, n = terrain_ref.ray_hfield(hf, origin, pnt[k], vec[k])
        if x < 0 or x > 2.0 - 1e-4:         # (at or below z = 0 the floor plane comes first or ties)
            continue
        assert g[k] == tg and abs(d[k] - x) < 2e-5, (k, d[k], x)
        np.testing.assert_allclose(nr[k], n, atol=1e-4)


def test_horizontal_rays_hit_a_risers_and_the_fields_sides(emu_t, bundled_only):
    hf = _stairs()
    env = _a1_on(hf)
    tg = env._model.ngeom - 1
    # the field: z = 0 on the centre platform (|x|, |y| <= 0.5), then steps 0.1 m down every 0.3 m to z = -0.5 at the
    # sides, base at z = -0.7. Rays: from inside the platform's solid outward along +x; from outside the field below its
    # edge along +x and +y (the sides); from outside above the edge along +x (a riser, between the steps at -0.2 and -0.3).
    # (From above, the floor plane at z = 0 hides every step of this field.)
    pnt = np.array([[0.0, 0.1, -0.05], [-3.0, 0.2, -0.6], [0.1, -3.0, -0.65], [-1.9, 0.13, -0.25]])
    vec = np.array([[1.0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [1.0, 0, 0]])
    d, g, nr = _emu_rays(emu_t, env, (0, 0), pnt, vec, flags=1)
    for k in range(len(pnt)):
        x, n = terrain_ref.ray_hfield(hf, (0, 0), pnt[k], vec[k])
        assert x >= 0 and g[k] == tg and abs(d[k] - x) < 2e-5, (k, d[k], x)
        np.testing.assert_allclose(nr[k], n, atol=1e-4)
    # the riser: the ray from inside the solid leaves it through the first step's face, between x = 0.5 and 0.55
    assert 0.5 - 1e-6 <= d[0] <= 0.55 + 1e-6
    # the sides: x = -rx (normal -x) and y = -ry (normal -y)
    assert abs(d[1] - (3.0 - hf.rx)) < 1e-5 and np.allclose(nr[1], [-1, 0, 0])
    assert abs(d[2] - (3.0 - hf.ry)) < 1e-5 and np.allclose(nr[2], [0, -1, 0])
    # the riser from outside: crossing z = -0.25 between x = -1.15 and -1.1, facing the ray
    assert -1.15 - 1e-5 <= -1.9 + d[3] <= -1.1 + 1e-5 and nr[3][0] < -0.5
    # no terrain without LS_RAY_STATIC, or with the world body excluded
    d2, g2, _ = _emu_rays(emu_t, env, (0, 0), pnt, vec, flags=2)
    assert np.all(g2 != tg)
    d3, g3, _ = _emu_rays(emu_t, env, (0, 0), pnt, vec, flags=3, exclude=0)
    assert np.all(g3 != tg)


# ---------------------------------------------------------------------------------------------------------------------
# 1b. the terrain unit's compiled figures (CUDA 12.9, the flags of __graft_entry__.NVCC_FLAGS): registers, stack frame,
#     spill stores, spill loads. The step kernels spill as UnitreeA1's own do (CfgEllEuler: 640 / 624 / 624-byte frames,
#     264 / 228 / 268 bytes of spill stores); the ray kernel spills nothing.
# ---------------------------------------------------------------------------------------------------------------------
TERRAIN_FIGURES = {
    "_ZN14locosimterrain11step_kernelINS_18CfgEllEulerTerrainEEEviNS_7DevTaskENS_10SolverOptsENS_11EngineStateEPKfPfS7_PhS7_iimliiPKhi": (128, 768, 324, 420),
    "_ZN14locosimterrain14substep_kernelINS_18CfgEllEulerTerrainEEEviNS_7DevTaskENS_10SolverOptsENS_11EngineStateEPKfPfS7_PhS7_iimliiPKhiiiNS_10SplitStateE": (128, 752, 292, 388),
    "_ZN14locosimterrain14persist_kernelINS_18CfgEllEulerTerrainEEEviNS_7DevTaskENS_10SolverOptsENS_11EngineStateEPKfPfS7_PhS7_iimliiPKhiNS_12PersistQueueE": (128, 752, 340, 336),
    "_ZN14locosimterrain12terrain_passINS_18CfgEllEulerTerrainEEEviRNS_4EnvSIT_EE": (None, 0, 112, 136),
    "_ZN14locosimterrain12terrain_passINS_9RoundLoopINS_18CfgEllEulerTerrainEEEEEviRNS_4EnvSIT_EE": (None, 0, 0, 0),
    "_ZN14locosimterrain10ray_kernelINS_9RoundLoopINS_18CfgEllEulerTerrainEEEEEviNS_11EngineStateENS_7RayArgsE": (150, 224, 0, 0),
}


def test_terrain_kernels_ptxas_figures(tmp_path):
    import subprocess
    from test_contact_list import NVCC, _nvcc_release, ptxas_figures
    if _nvcc_release() != "12.9":
        pytest.skip("the recorded figures are CUDA 12.9's")
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-prec-div=false",
             "-prec-sqrt=false", "-ftz=true", "-Xptxas", "-v", "-cubin"]
    src = os.path.join(ROOT, "loco_mujoco_b200", "csrc", "locosim_terrain.cu")
    p = subprocess.run([NVCC] + flags + ["-o", str(tmp_path / "t.cubin"), src], capture_output=True, text=True)
    assert p.returncode == 0, (p.stdout + p.stderr)[-3000:]
    now = ptxas_figures(p.stdout + p.stderr)
    assert {k: now.get(k) for k in TERRAIN_FIGURES} == TERRAIN_FIGURES
