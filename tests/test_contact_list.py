"""Contact list (MuJoCo's d.contact with each contact's mj_contactForce, include/locosim.h locosim_set_contact_list_outputs)
without a GPU: the header constants, the host-side rules, the serial build of the CUDA core on hand-built scenes and against
the fp64 reference's last sub-step, and the compiled step kernels' register budget."""
import os
import re
import shutil
import subprocess
import tempfile
import types

import numpy as np
import pytest

import contact_list_ref as clr
import contact_wrench_ref as cwr
from full_body import make_variant
from helpers import ROOT, blobs, make_env

p = cwr._p


@pytest.fixture(scope="module")
def ref():
    return cwr.load()


def _compile(xml):
    from loco_mujoco_b200 import mjcf, modelpack
    with tempfile.NamedTemporaryFile("w", suffix=".xml", delete=False) as f:
        f.write(xml)
        path = f.name
    try:
        m = mjcf.compile_model(mjcf.XmlHandle(path), fuse_static=False)
    finally:
        os.unlink(path)
    ints, reals = modelpack.pack(m)
    return m, (np.ascontiguousarray(ints, dtype=np.int32), np.ascontiguousarray(reals, dtype=np.float64))


class _EmuList:
    """the serial core of a compiled model with the contact list registered (row 0 of the engine's layout)"""

    def __init__(self, emu, packed, register=True):
        clr.emu_bind(emu)
        self.emu, self.ints, self.reals = emu, packed[0], packed[1]
        self.s = emu.emu_create(p(self.ints), len(self.ints), p(self.reals), len(self.reals))
        assert self.s
        self.C = emu.emu_max_contacts(self.s)
        self.ncon = np.full(1, -7, dtype=np.int32)
        self.con = np.full((self.C, clr.DIM), np.nan, dtype=np.float32)
        self.con_id = np.full((self.C, clr.ID_DIM), -7, dtype=np.int32)
        if register:
            emu.emu_set_contact_list(self.s, p(self.ncon), p(self.con), p(self.con_id))

    def step(self, q, v, ctrl, nsub, ws=None):
        self.emu.emu_reset(self.s, p(np.ascontiguousarray(q, dtype=np.float64)), p(np.ascontiguousarray(v, dtype=np.float64)))
        self.emu.emu_set_ws(self.s, p(np.ascontiguousarray(np.zeros(len(q)) if ws is None else ws, dtype=np.float64)))
        self.emu.emu_step(self.s, p(np.ascontiguousarray(ctrl, dtype=np.float64)), int(nsub))
        return clr.unpack(self.ncon[0], self.con, self.con_id)

    def state(self, nv):
        q, v, w = np.zeros(nv), np.zeros(nv), np.zeros(nv)
        self.emu.emu_get_state(self.s, p(q), p(v))
        self.emu.emu_get_ws(self.s, p(w))
        return q, v, w

    def close(self):
        self.emu.emu_destroy(self.s)


def _settle(ref, packed, nv, q0, n=400):
    import ctypes
    lib = ref.lib
    sim = ctypes.c_void_p(lib.ref_create(p(packed[0]), len(packed[0]), p(packed[1]), len(packed[1])))
    lib.ref_reset(sim, p(np.ascontiguousarray(q0, dtype=np.float64)), p(np.zeros(nv)))
    for _ in range(n):
        lib.ref_step(sim, None, 1)
    q, v = np.zeros(nv), np.zeros(nv)
    lib.ref_get_state(sim, p(q), p(v))
    lib.ref_destroy(sim)
    return q, v


# ---------------------------------------------------------------------------------------------------------------------
# hand-built scenes (serial core)
# ---------------------------------------------------------------------------------------------------------------------
BOX_XML = """
<mujoco model="box">
  <option timestep="0.002" integrator="Euler" cone="pyramidal"/>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 1" condim="3"/>
    <body name="box" pos="0.5 -0.25 0.2">
      <joint name="x" type="slide" axis="1 0 0"/><joint name="y" type="slide" axis="0 1 0"/>
      <joint name="z" type="slide" axis="0 0 1"/>
      <geom name="g" type="box" size="0.1 0.08 0.05" pos="0 0 -0.15" mass="4" condim="3"/>
    </body>
  </worldbody>
</mujoco>
"""
BALL_XML = """
<mujoco model="ball">
  <option timestep="0.002" integrator="Euler" cone="{cone}"/>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 1" condim="{condim}" friction="1 0.05 0.001"/>
    <body name="ball" pos="0.3 0.2 0.1">
      <joint name="z" type="slide" axis="0 0 1"/><joint name="spin" type="hinge" axis="0 0 1"/>
      <geom name="g" type="sphere" size="0.1" mass="2" condim="{condim}" friction="1 0.05 0.001"/>
    </body>
  </worldbody>
</mujoco>
"""


def test_box_at_rest_has_four_corner_contacts(emu, ref):
    m, packed = _compile(BOX_XML)
    q, v = _settle(ref, packed, m.nv, np.zeros(3))
    assert np.abs(v).max() < 1e-6
    e = _EmuList(emu, packed)
    got = e.step(q, v, np.zeros(1), 5)
    W = 4 * 9.81
    assert len(got["dist"]) == 4 and clr.empty_rows_ok(e.ncon[0], e.con, e.con_id)
    assert np.array_equal(got["geom"], [[0, 1]] * 4) and np.array_equal(got["body"], [[0, 1]] * 4)
    assert np.array_equal(got["dim"], [3] * 4)
    assert np.allclose(got["frame"][:, 0:3], [0, 0, 1], atol=1e-6)                     # n: floor -> box, up
    assert np.allclose(got["force"][:, 0].sum(), W, rtol=1e-3)                          # the weight
    assert np.allclose(got["force"][:, 0], W / 4, rtol=2e-2)                            # a quarter at each corner
    assert np.abs(got["force"][:, 1:]).max() < 1e-3 * W                                 # no friction at rest
    centre = np.array([0.5 + q[0], -0.25 + q[1]])
    corners = {(sx, sy) for sx in (-1, 1) for sy in (-1, 1)}
    seen = {(int(np.sign(x - centre[0])), int(np.sign(y - centre[1]))) for x, y in got["pos"][:, :2]}
    assert seen == corners
    assert np.allclose(np.abs(got["pos"][:, :2] - centre), [0.1, 0.08], atol=1e-5)
    # each position is the midpoint of its corner's penetration: z = dist / 2 on the plane z = 0
    assert np.all(got["dist"] < 0) and np.allclose(got["pos"][:, 2], got["dist"] / 2, atol=1e-6)
    e.close()


@pytest.mark.parametrize("cone", ["pyramidal", "elliptic"])
def test_sphere_with_a_known_penetration(emu, cone):
    """one sub-step from rest at centre height 0.09: the list is the sub-step's start state, dist = 0.09 - r and the
    position the midpoint of the penetration below the centre"""
    m, packed = _compile(BALL_XML.format(cone=cone, condim=3))
    e = _EmuList(emu, packed)
    got = e.step(np.array([-0.01, 0.0]), np.zeros(2), np.zeros(1), 1)
    assert len(got["dist"]) == 1 and np.array_equal(got["geom"], [[0, 1]]) and got["dim"][0] == 3
    assert abs(got["dist"][0] - (-0.01)) < 1e-6
    assert np.allclose(got["pos"][0], [0.3, 0.2, -0.005], atol=1e-6)
    assert np.allclose(got["frame"][0, :3], [0, 0, 1], atol=1e-7)
    fr = got["frame"][0].reshape(3, 3)
    assert np.allclose(fr @ fr.T, np.eye(3), atol=1e-6)                                  # an orthonormal frame
    assert got["force"][0, 0] > 0 and np.array_equal(got["force"][0, 3:], np.zeros(3))   # components past dim are 0
    e.close()


def test_spinning_sphere_torsion_opposes_the_spin(emu, ref):
    m, packed = _compile(BALL_XML.format(cone="elliptic", condim=6))
    q, _ = _settle(ref, packed, m.nv, np.zeros(2))
    e = _EmuList(emu, packed)
    W = 2 * 9.81
    for spin in (1.0, -1.0):
        got = e.step(q, [0.0, spin], np.zeros(1), 5)
        assert len(got["dist"]) == 1 and got["dim"][0] == 6
        f = got["force"][0]
        assert np.allclose(f[0], W, rtol=0.05), f
        assert np.sign(f[3]) == -np.sign(spin) and 0.01 * W * 0.05 < abs(f[3]) <= 1.01 * 0.05 * W, (spin, f)
    e.close()


# ---------------------------------------------------------------------------------------------------------------------
# the serial core against the fp64 reference's last sub-step
# ---------------------------------------------------------------------------------------------------------------------
TASKS = ["UnitreeA1.simple", "HumanoidTorque.run", "Talos.walk", "Atlas.walk+arms+back", "Talos.walk+arms"]


@pytest.mark.parametrize("task", TASKS)
def test_serial_core_matches_the_reference(emu, ref, bundled_only, task):
    """One control step from reset-table states under random actions: the serial build of the CUDA core (same source as the
    kernels) against the oracle's last sub-step, contact by contact in list order, within clr.TOL; where the oracle's own list
    changes under an fp32-sized perturbation of the start state (a contact switching within the step), within 10x that."""
    from loco_mujoco_b200 import modelpack
    env = make_variant(task)
    m, spec = env._model, env.task_spec()
    mb, tb = blobs(env)
    ints, reals = [np.ascontiguousarray(x) for x in modelpack.pack(m)]
    e = _EmuList(emu, (ints.astype(np.int32), reals.astype(np.float64)))
    assert e.C == 16
    rng = np.random.RandomState(11)
    table = spec.table.reshape(-1, spec.table.shape[-1])
    user = env._model_user_features[0]
    touched, allowed = 0, 0
    for i in rng.randint(len(table), size=8):
        oe = ref.env(mb, tb)
        oe.set_user(user)
        oe.reset_to(i // spec.table.shape[1], i % spec.table.shape[1])
        q, v = oe.get_state()
        a = rng.uniform(-1, 1, m.nu)
        ctrl = np.zeros(m.nu)
        ctrl[spec.act_idx] = a * spec.act_delta + spec.act_mean
        got = e.step(q, v, ctrl, spec.n_substeps)
        cwr.env_step(ref, oe, a)
        want = clr.reference(ref, oe.sim, m)
        oe.close()
        assert clr.empty_rows_ok(e.ncon[0], e.con, e.con_id)
        touched += int(len(want["dist"]) > 0 and np.abs(want["force"]).max() > 1.0)
        err = clr.mismatch(got, want)
        if err > 1.0:
            gap = clr.sensitivity(ref, mb, tb, m, q, v, a, want, user=user)
            assert err < 10 * gap, (task, i, err, gap)
            allowed += 1
    e.close()
    assert touched >= 4, "too few states with contact forces"
    assert allowed <= 2, allowed


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "HumanoidTorque.run"])
def test_registering_changes_no_other_bit(emu, bundled_only, task):
    """the serial core's state, warm start, contact outputs and dof outputs are the same bit for bit with and without the
    list registered; and with the other outputs registered the list is the same as alone (EnvS::substep advances once per
    sub-step whichever outputs are registered)"""
    from loco_mujoco_b200 import modelpack
    cwr.emu_bind(emu)
    emu.emu_set_dof.restype = None
    emu.emu_set_dof.argtypes = [emu.emu_set_contact.argtypes[0]] * 2
    env = make_env(task)
    m, spec = env._model, env.task_spec()
    ints, reals = [np.ascontiguousarray(x) for x in modelpack.pack(m)]
    packed = (ints.astype(np.int32), reals.astype(np.float64))
    table = spec.table.reshape(-1, spec.table.shape[-1])
    rng = np.random.RandomState(5)
    runs = {}
    for register, others in ((False, False), (True, False), (False, True), (True, True)):
        e = _EmuList(emu, packed, register=register)
        wrench = np.zeros((m.nbody, 6), dtype=np.float32)
        dof = np.zeros((m.nv, 3), dtype=np.float32)
        if others:
            emu.emu_set_contact(e.s, p(wrench))
            emu.emu_set_dof(e.s, p(dof))
        rng.seed(5)
        out = []
        for i in rng.randint(len(table), size=4):
            q, v = table[i, :m.nv], table[i, m.nv:2 * m.nv]
            ctrl = np.zeros(m.nu)
            ctrl[spec.act_idx] = rng.uniform(-1, 1, m.nu) * spec.act_delta + spec.act_mean
            got = e.step(q, v, ctrl, spec.n_substeps)
            out.append((e.state(m.nv), wrench.copy(), dof.copy(), got if register else None))
        runs[(register, others)] = out
        e.close()
    for others in (False, True):
        for (s0, w0, d0, _), (s1, w1, d1, _) in zip(runs[(False, others)], runs[(True, others)]):
            assert all(np.array_equal(a, b) for a, b in zip(s0, s1))
            assert np.array_equal(w0, w1) and np.array_equal(d0, d1)
    assert any(np.abs(w).max() > 0 for _, w, _, _ in runs[(True, True)])
    for (_, _, _, a), (_, _, _, b) in zip(runs[(True, False)], runs[(True, True)]):
        assert len(a["dist"]) > 0 or len(b["dist"]) == 0
        assert all(np.array_equal(a[k], b[k]) for k in a)


# ---------------------------------------------------------------------------------------------------------------------
# header and host logic
# ---------------------------------------------------------------------------------------------------------------------
def test_header_constants_match_the_package(tmp_path):
    from loco_mujoco_b200 import engine
    src = tmp_path / "conlist.c"
    src.write_text('#include <stdio.h>\n#include "locosim.h"\nint main(void) {\n'
                   '  printf("%d %d %d %d %d %d %d %d %d %d %d\\n", LS_CONLIST_DIM, LS_CONLIST_DIST, LS_CONLIST_POS,'
                   " LS_CONLIST_FRAME, LS_CONLIST_FORCE, LS_CONLIST_ID_DIM, LS_CONLIST_GEOM1, LS_CONLIST_GEOM2,"
                   " LS_CONLIST_BODY1, LS_CONLIST_BODY2, LS_CONLIST_CONDIM);\n  return 0; }\n")
    exe = tmp_path / "conlist"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    v = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    F, I = engine.CONLIST_COLUMNS, engine.CONLIST_ID_COLUMNS
    assert v == [engine.CONLIST_DIM, F["dist"][0], F["pos"][0], F["frame"][0], F["force"][0], engine.CONLIST_ID_DIM,
                 I["geom"][0], I["geom"][0] + 1, I["body"][0], I["body"][0] + 1, I["dim"][0]]
    # the columns tile the rows
    for cols, dim in ((F, engine.CONLIST_DIM), (I, engine.CONLIST_ID_DIM)):
        spans = sorted(cols.values())
        assert spans[0][0] == 0 and sum(n for _, n in spans) == dim
        assert all(a + n == b for (a, n), (b, _) in zip(spans, spans[1:]))


def _fake_engine(monkeypatch, calls):
    import torch
    from loco_mujoco_b200 import engine as engine_mod
    eng = object.__new__(engine_mod.CudaEngine)
    eng.torch = torch
    eng.n_envs, eng.max_contacts, eng.device, eng.h = 4, 16, torch.device("cpu"), None
    eng._conlist_out = (None, None, None)
    eng.lib = types.SimpleNamespace(locosim_set_contact_list_outputs=lambda h, a, b, c: calls.append((a, b, c)) or 0)
    monkeypatch.setattr(engine_mod, "_ptr", lambda t: None if t is None else t.data_ptr())
    return eng


def test_set_contact_list_outputs_validates_its_arguments(monkeypatch):
    """all or none, dtypes, shapes, contiguity, device and overlap are checked before the engine is called"""
    import torch
    calls = []
    eng = _fake_engine(monkeypatch, calls)
    n = torch.zeros(4, dtype=torch.int32)
    c = torch.zeros((4, 16, 19), dtype=torch.float32)
    i = torch.zeros((4, 16, 5), dtype=torch.int32)
    eng.set_contact_list_outputs(n, c, i)
    assert calls == [(n.data_ptr(), c.data_ptr(), i.data_ptr())] and eng._conlist_out == (n, c, i)
    eng.set_contact_list_outputs()
    assert calls[-1] == (None, None, None) and eng._conlist_out == (None, None, None)
    big = torch.zeros(4 + 4 * 16 * 19 + 4 * 16 * 5, dtype=torch.int32)
    bad = [(n, c, None), (None, c, i), (n, None, None),                                  # all or none
           (n.float(), c, i), (n, c.double(), i), (n, c, i.float()), (n, c.int(), i),      # dtypes
           (torch.zeros(5, dtype=torch.int32), c, i), (n, torch.zeros((4, 16, 13)), i),    # shapes
           (n, c, torch.zeros((4, 15, 5), dtype=torch.int32)), (n, torch.zeros((4, 32, 19)), i),
           (n, torch.zeros((4, 19, 16)).transpose(1, 2), i),                              # contiguity
           (n, c, i.numpy()),                                                             # not a tensor
           (big[:4], big[4:4 + 4 * 16 * 19].view(torch.float32).view(4, 16, 19), big[:320].view(4, 16, 5)),   # overlap
           (big[:4], big[:4 * 16 * 19].view(torch.float32).view(4, 16, 19), big[-320:].view(4, 16, 5))]
    for b in bad:
        with pytest.raises(ValueError):
            eng.set_contact_list_outputs(*b)
    assert len(calls) == 2
    eng.device = torch.device("cuda", 0)                                                 # another device
    with pytest.raises(ValueError):
        eng.set_contact_list_outputs(n, c, i)
    assert len(calls) == 2


class _RecordingEngine:
    """Stands in for CudaEngine on a CPU-only box: records what the env registers."""

    def __init__(self, model_blobs, task_blobs, n_envs, device=0, **kw):
        import torch
        self.device, self.n_envs, self.max_contacts, self.calls = torch.device("cpu"), n_envs, 16, []

    def set_contact_list_outputs(self, ncon=None, con=None, con_id=None):
        self.calls.append((ncon, con, con_id))

    def set_param_pool(self, pool):
        pass

    def close(self):
        pass


def test_contacts_are_lazy_and_survive_an_engine_rebuild(bundled_only, monkeypatch):
    import torch
    from loco_mujoco_b200 import engine as engine_mod
    monkeypatch.setattr(engine_mod, "CudaEngine", _RecordingEngine)
    env = make_env("UnitreeA1.simple", num_envs=5)
    eng = env._get_engine()
    assert eng.calls == []                                       # nothing registered until the list is asked for
    c = env.contacts
    assert len(eng.calls) == 1 and env.contacts is c and len(eng.calls) == 1
    ncon, con, con_id = eng.calls[0]
    assert c.ncon is ncon and str(ncon.dtype) == str(con_id.dtype) == "torch.int32"
    assert tuple(con.shape) == (5, 16, 19) and tuple(con_id.shape) == (5, 16, 5) and str(con.dtype) == "torch.float32"
    assert float(con.abs().max()) == 0.0 and int(con_id.max()) == -1 and int(ncon.abs().max()) == 0
    shapes = dict(ncon=(5,), dist=(5, 16), pos=(5, 16, 3), frame=(5, 16, 3, 3), force=(5, 16, 6), geom=(5, 16, 2),
                  body=(5, 16, 2), dim=(5, 16))
    assert {k: tuple(getattr(c, k).shape) for k in shapes} == shapes
    # the views are views of the registered buffers, at the header's columns
    con.copy_(torch.arange(con.numel(), dtype=con.dtype).view(con.shape))
    con_id.copy_(torch.arange(con_id.numel(), dtype=con_id.dtype).view(con_id.shape))
    assert float(c.dist[1, 2]) == float(con[1, 2, 0]) and float(c.frame[1, 2, 1, 0]) == float(con[1, 2, 7])
    assert float(c.force[1, 2, 5]) == float(con[1, 2, 18]) and float(c.pos[0, 3, 2]) == float(con[0, 3, 3])
    assert int(c.geom[1, 2, 1]) == int(con_id[1, 2, 1]) and int(c.body[1, 2, 0]) == int(con_id[1, 2, 2])
    assert int(c.dim[1, 2]) == int(con_id[1, 2, 4])
    env.set_launch_geometry(4)                                   # rebuilds the engine: the same tensors are registered again
    eng2 = env._get_engine()
    assert eng2 is not eng and len(eng2.calls) == 1 and all(a is b for a, b in zip(eng2.calls[0], (ncon, con, con_id)))


def test_geom_index_and_names(bundled_only):
    env = make_env("UnitreeA1.simple", num_envs=2)
    names = env.geom_names
    assert len(names) == env._model.ngeom
    for g, name in enumerate(names):
        if name is not None and names.count(name) == 1:
            assert env.geom_index(name) == g
    with pytest.raises(ValueError):
        env.geom_index("no such geom")
    with pytest.raises(ValueError):
        env.geom_index(None)


def test_4ages_all_refuses_the_contact_list(bundled_only):
    from loco_mujoco_b200 import LocoEnv
    env = LocoEnv.make("HumanoidTorque4Ages.walk.all.real", num_envs=8, debug=True)
    for f in (lambda: env.contacts, lambda: env.geom_names, lambda: env.geom_index("floor")):
        with pytest.raises(NotImplementedError):
            f()


# ---------------------------------------------------------------------------------------------------------------------
# register budget: compiling the writer into the step kernels moves no kernel's figures
# ---------------------------------------------------------------------------------------------------------------------
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def _nvcc_release():
    try:
        out = subprocess.run([NVCC, "--version"], capture_output=True, text=True).stdout
    except OSError:
        return None
    m = re.search(r"release (\d+\.\d+)", out)
    return m.group(1) if m else None


def ptxas_figures(text):
    """{function: (registers or None, stack frame, spill stores, spill loads)} of an -Xptxas -v log"""
    out, name = {}, None
    for line in text.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            out[name] = [None, int(m.group(1)), int(m.group(2)), int(m.group(3))]
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and name in out and out[name][0] is None:
            out[name][0] = int(m.group(1))
            name = None
    return {k: tuple(v) for k, v in out.items()}


# What the parent commit's sources compile to with CUDA 12.9's nvcc (the flags of __graft_entry__.NVCC_FLAGS, device code):
# per translation unit, every kernel's registers and every kernel's and __noinline__ function's stack frame, spill stores
# and spill loads, as "registers stack stores loads name" ("-" for a function that is not a kernel).
PARENT_FIGURES = {
    "locosim.cu": """
- 0 0 0 _Z10chol_solveILi18ELi19EEvPAT0__fPf
- 0 0 0 _Z10chol_solveILi19ELi20EEvPAT0__fPf
- 0 0 0 _Z10chol_solveILi29ELi30EEvPAT0__fPf
- 0 0 0 _Z10convex_jobI11CfgEllEulerEviRK4EnvSIT_ERS3_iPf
- 0 0 0 _Z10convex_jobI11CfgPyrEulerEviRK4EnvSIT_ERS3_iPf
- 0 0 0 _Z10convex_jobI13CfgPyrEuler29EviRK4EnvSIT_ERS3_iPf
- 0 0 0 _Z10convex_jobI9CfgPyrRK4EviRK4EnvSIT_ERS3_iPf
- 0 0 0 _Z10convex_jobI9RoundLoopI11CfgEllEulerEEviRK4EnvSIT_ERS5_iPf
- 0 0 0 _Z10convex_jobI9RoundLoopI11CfgPyrEulerEEviRK4EnvSIT_ERS5_iPf
- 0 0 0 _Z10convex_jobI9RoundLoopI13CfgPyrEuler29EEviRK4EnvSIT_ERS5_iPf
- 0 0 0 _Z10convex_jobI9RoundLoopI9CfgPyrRK4EEviRK4EnvSIT_ERS5_iPf
- 0 0 12 _Z10crb_factorI11CfgEllEulerEviR4EnvSIT_E
- 0 0 12 _Z10crb_factorI11CfgPyrEulerEviR4EnvSIT_E
- 0 0 12 _Z10crb_factorI13CfgPyrEuler29EviR4EnvSIT_E
- 0 0 12 _Z10crb_factorI9CfgPyrRK4EviR4EnvSIT_E
- 0 0 0 _Z10crb_factorI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E
- 0 0 0 _Z10crb_factorI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E
- 0 0 0 _Z10crb_factorI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E
- 0 0 0 _Z10crb_factorI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E
- 0 0 0 _Z10euler_stepI11CfgEllEulerEviR4EnvSIT_E
- 0 0 0 _Z10euler_stepI11CfgPyrEulerEviR4EnvSIT_E
- 0 0 0 _Z10euler_stepI13CfgPyrEuler29EviR4EnvSIT_E
- 0 0 0 _Z10kinematicsI11CfgEllEulerEviR4EnvSIT_E
- 0 0 0 _Z10kinematicsI11CfgPyrEulerEviR4EnvSIT_E
- 0 0 0 _Z10kinematicsI13CfgPyrEuler29EviR4EnvSIT_E
- 0 0 0 _Z10kinematicsI9CfgPyrRK4EviR4EnvSIT_E
- 0 0 0 _Z10kinematicsI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E
- 0 0 0 _Z10kinematicsI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E
- 0 0 0 _Z10kinematicsI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E
- 0 0 0 _Z10kinematicsI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E
- 0 0 0 _Z10ls_prepareI11CfgEllEulerEviR4EnvSIT_E
- 0 0 0 _Z10ls_prepareI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E
- 0 0 0 _Z10plane_meshP6RawConfPKfS2_S2_S2_S2_if
- 0 0 0 _Z10sphere_boxP6RawConfPKffS2_S2_S2_
72 56 0 0 _Z11body_kernelI11CfgEllEulerEvi7DevTask11EngineStatePKhS4_iimlPK4int2
72 56 0 0 _Z11body_kernelI11CfgPyrEulerEvi7DevTask11EngineStatePKhS4_iimlPK4int2
71 56 0 0 _Z11body_kernelI13CfgPyrEuler29Evi7DevTask11EngineStatePKhS4_iimlPK4int2
71 56 0 0 _Z11body_kernelI9CfgPyrRK4Evi7DevTask11EngineStatePKhS4_iimlPK4int2
- 0 0 0 _Z11chol_factorILi18ELi19EEviPAT0__f
- 0 0 0 _Z11chol_factorILi19ELi20EEviPAT0__f
- 0 0 0 _Z11chol_factorILi29ELi30EEviPAT0__f
- 0 0 0 _Z11dof_outputsI11CfgEllEulerEviR4EnvSIT_E
- 0 0 0 _Z11dof_outputsI11CfgPyrEulerEviR4EnvSIT_E
- 0 0 0 _Z11dof_outputsI13CfgPyrEuler29EviR4EnvSIT_E
- 0 0 0 _Z11dof_outputsI9CfgPyrRK4EviR4EnvSIT_E
- 0 0 0 _Z11line_searchI11CfgEllEulerEfiR4EnvSIT_E10SolverOptsfff
- 0 0 0 _Z11line_searchI11CfgPyrEulerEfiR4EnvSIT_E10SolverOptsfff
- 0 0 0 _Z11line_searchI13CfgPyrEuler29EfiR4EnvSIT_E10SolverOptsfff
- 0 0 0 _Z11line_searchI9CfgPyrRK4EfiR4EnvSIT_E10SolverOptsfff
- 0 0 0 _Z11line_searchI9RoundLoopI11CfgEllEulerEEfiR4EnvSIT_E10SolverOptsfff
- 0 0 0 _Z11line_searchI9RoundLoopI11CfgPyrEulerEEfiR4EnvSIT_E10SolverOptsfff
- 0 0 0 _Z11line_searchI9RoundLoopI13CfgPyrEuler29EEfiR4EnvSIT_E10SolverOptsfff
- 0 0 0 _Z11line_searchI9RoundLoopI9CfgPyrRK4EEfiR4EnvSIT_E10SolverOptsfff
- 0 0 0 _Z11pair_narrowI11CfgEllEulerEiiR4EnvSIT_EiP6RawConPiS7_Pf
- 0 0 0 _Z11pair_narrowI11CfgPyrEulerEiiR4EnvSIT_EiP6RawConPiS7_Pf
- 0 0 0 _Z11pair_narrowI13CfgPyrEuler29EiiR4EnvSIT_EiP6RawConPiS7_Pf
- 0 0 0 _Z11pair_narrowI9CfgPyrRK4EiiR4EnvSIT_EiP6RawConPiS7_Pf
- 0 0 0 _Z11pair_narrowI9RoundLoopI11CfgEllEulerEEiiR4EnvSIT_EiP6RawConPiS9_Pf
- 0 0 0 _Z11pair_narrowI9RoundLoopI11CfgPyrEulerEEiiR4EnvSIT_EiP6RawConPiS9_Pf
- 0 0 0 _Z11pair_narrowI9RoundLoopI13CfgPyrEuler29EEiiR4EnvSIT_EiP6RawConPiS9_Pf
- 0 0 0 _Z11pair_narrowI9RoundLoopI9CfgPyrRK4EEiiR4EnvSIT_EiP6RawConPiS9_Pf
14 0 0 0 _Z11rank_kernelPKiPiii
128 640 264 400 _Z11step_kernelI11CfgEllEulerEvi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhi
128 640 264 400 _Z11step_kernelI11CfgPyrEulerEvi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhi
128 720 264 400 _Z11step_kernelI13CfgPyrEuler29Evi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhi
128 752 312 400 _Z11step_kernelI9CfgPyrRK4Evi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhi
- 0 0 0 _Z12body_outputsI11CfgEllEulerEviR4EnvSIT_EPfS5_
- 0 0 0 _Z12body_outputsI11CfgPyrEulerEviR4EnvSIT_EPfS5_
- 0 0 0 _Z12body_outputsI13CfgPyrEuler29EviR4EnvSIT_EPfS5_
- 0 0 0 _Z12body_outputsI9CfgPyrRK4EviR4EnvSIT_EPfS5_
- 0 0 0 _Z12fill_contactI11CfgEllEulerEviR4EnvSIT_EiiifPK6RawCon
- 0 0 0 _Z12fill_contactI11CfgPyrEulerEviR4EnvSIT_EiiifPK6RawCon
- 0 0 0 _Z12fill_contactI13CfgPyrEuler29EviR4EnvSIT_EiiifPK6RawCon
- 0 0 0 _Z12fill_contactI9CfgPyrRK4EviR4EnvSIT_EiiifPK6RawCon
- 0 0 0 _Z12fill_contactI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_EiiifPK6RawCon
- 0 0 0 _Z12fill_contactI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_EiiifPK6RawCon
- 0 0 0 _Z12fill_contactI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_EiiifPK6RawCon
- 0 0 0 _Z12fill_contactI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_EiiifPK6RawCon
- 0 0 0 _Z12impedance_KBPKfS0_fffPfS1_S1_
- 0 0 0 _Z12passive_biasI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E
- 0 0 0 _Z12passive_biasI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E
- 0 0 0 _Z12passive_biasI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E
- 0 0 0 _Z12passive_biasI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E
- 0 0 0 _Z12plane_sphereP6RawConfPKfS2_S2_f
32 32 0 0 _Z12reset_kerneli7DevTask11EngineStatePKhPKiS4_S4_PfimlP4int2
- 0 0 0 _Z13plane_capsuleP6RawConfPKfS2_S2_S2_S2_
- 0 0 12 _Z13smooth_forcesI11CfgEllEulerEviR4EnvSIT_E
- 0 0 12 _Z13smooth_forcesI11CfgPyrEulerEviR4EnvSIT_E
- 0 0 12 _Z13smooth_forcesI13CfgPyrEuler29EviR4EnvSIT_E
- 0 0 12 _Z13smooth_forcesI9CfgPyrRK4EviR4EnvSIT_E
- 0 0 0 _Z13smooth_forcesI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E
- 0 0 0 _Z13smooth_forcesI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E
- 0 0 0 _Z13smooth_forcesI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E
- 0 0 0 _Z13smooth_forcesI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E
- 0 0 0 _Z14contact_forcesI11CfgEllEulerEviR4EnvSIT_EPKii
- 0 0 0 _Z14contact_forcesI11CfgPyrEulerEviR4EnvSIT_EPKii
- 0 0 0 _Z14contact_forcesI13CfgPyrEuler29EviR4EnvSIT_EPKii
- 0 0 0 _Z14contact_forcesI9CfgPyrRK4EviR4EnvSIT_EPKii
- 0 0 0 _Z14contact_wrenchI11CfgEllEulerEviR4EnvSIT_E
- 0 0 0 _Z14contact_wrenchI11CfgPyrEulerEviR4EnvSIT_E
- 0 0 0 _Z14contact_wrenchI13CfgPyrEuler29EviR4EnvSIT_E
- 0 0 0 _Z14contact_wrenchI9CfgPyrRK4EviR4EnvSIT_E
- 0 0 0 _Z14convex_consumeI11CfgEllEulerEviR4EnvSIT_EiPKf
- 0 0 0 _Z14convex_consumeI11CfgPyrEulerEviR4EnvSIT_EiPKf
- 0 0 0 _Z14convex_consumeI13CfgPyrEuler29EviR4EnvSIT_EiPKf
- 0 0 0 _Z14convex_consumeI9CfgPyrRK4EviR4EnvSIT_EiPKf
- 0 0 0 _Z14convex_consumeI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_EiPKf
- 0 0 0 _Z14convex_consumeI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_EiPKf
- 0 0 0 _Z14convex_consumeI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_EiPKf
- 0 0 0 _Z14convex_consumeI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_EiPKf
- 0 0 0 _Z14dynamics_termsI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E6DynOut
- 0 0 0 _Z14dynamics_termsI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E6DynOut
- 0 0 0 _Z14dynamics_termsI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E6DynOut
- 0 0 0 _Z14dynamics_termsI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E6DynOut
128 320 0 0 _Z14forward_kernelI9RoundLoopI11CfgEllEulerEEvi11EngineState7DevTaskPKi10SolverOptsPKf6FwdOut
128 320 0 0 _Z14forward_kernelI9RoundLoopI11CfgPyrEulerEEvi11EngineState7DevTaskPKi10SolverOptsPKf6FwdOut
128 400 0 0 _Z14forward_kernelI9RoundLoopI13CfgPyrEuler29EEvi11EngineState7DevTaskPKi10SolverOptsPKf6FwdOut
128 400 0 0 _Z14forward_kernelI9RoundLoopI9CfgPyrRK4EEvi11EngineState7DevTaskPKi10SolverOptsPKf6FwdOut
- 0 0 32 _Z14fwd_constraintI11CfgEllEulerEviR4EnvSIT_E10SolverOpts
- 0 0 32 _Z14fwd_constraintI11CfgPyrEulerEviR4EnvSIT_E10SolverOpts
- 0 0 32 _Z14fwd_constraintI13CfgPyrEuler29EviR4EnvSIT_E10SolverOpts
- 0 0 36 _Z14fwd_constraintI9CfgPyrRK4EviR4EnvSIT_E10SolverOpts
- 0 0 0 _Z14fwd_constraintI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E10SolverOpts
- 0 0 0 _Z14fwd_constraintI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E10SolverOpts
- 0 0 0 _Z14fwd_constraintI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E10SolverOpts
- 0 0 0 _Z14fwd_constraintI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E10SolverOpts
- 0 0 0 _Z14init_workspaceI11CfgEllEulerEviR4EnvSIT_E
- 0 0 0 _Z14init_workspaceI11CfgPyrEulerEviR4EnvSIT_E
- 0 0 0 _Z14init_workspaceI13CfgPyrEuler29EviR4EnvSIT_E
- 0 0 0 _Z14init_workspaceI9CfgPyrRK4EviR4EnvSIT_E
- 0 0 0 _Z14init_workspaceI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E
- 0 0 0 _Z14init_workspaceI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E
- 0 0 0 _Z14init_workspaceI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E
- 0 0 0 _Z14init_workspaceI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E
124 320 0 0 _Z14inverse_kernelI9RoundLoopI11CfgEllEulerEEvi11EngineState7DevTaskPKiPKfS8_fPf
124 320 0 0 _Z14inverse_kernelI9RoundLoopI11CfgPyrEulerEEvi11EngineState7DevTaskPKiPKfS8_fPf
124 400 0 0 _Z14inverse_kernelI9RoundLoopI13CfgPyrEuler29EEvi11EngineState7DevTaskPKiPKfS8_fPf
124 400 0 0 _Z14inverse_kernelI9RoundLoopI9CfgPyrRK4EEvi11EngineState7DevTaskPKiPKfS8_fPf
128 624 268 328 _Z14persist_kernelI11CfgEllEulerEvi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhi12PersistQueue
128 624 268 328 _Z14persist_kernelI11CfgPyrEulerEvi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhi12PersistQueue
128 704 268 328 _Z14persist_kernelI13CfgPyrEuler29Evi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhi12PersistQueue
128 752 332 328 _Z14persist_kernelI9CfgPyrRK4Evi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhi12PersistQueue
- 0 0 0 _Z14plane_cylinderP6RawConfPKfS2_S2_S2_S2_
- 0 0 0 _Z14sphere_capsuleP6RawConfPKffS2_S2_S2_
128 624 228 348 _Z14substep_kernelI11CfgEllEulerEvi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhiii10SplitState
128 624 228 348 _Z14substep_kernelI11CfgPyrEulerEvi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhiii10SplitState
128 704 228 348 _Z14substep_kernelI13CfgPyrEuler29Evi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhiii10SplitState
128 752 284 364 _Z14substep_kernelI9CfgPyrRK4Evi7DevTask10SolverOpts11EngineStatePKfPfS6_PhS6_iimliiPKhiii10SplitState
- 0 0 0 _Z15capsule_capsuleP6RawConfPKfS2_S2_S2_S2_S2_
64 32 0 0 _Z15dynamics_kernelI9RoundLoopI11CfgEllEulerEEvi11EngineState6DynOut
64 32 0 0 _Z15dynamics_kernelI9RoundLoopI11CfgPyrEulerEEvi11EngineState6DynOut
64 32 0 0 _Z15dynamics_kernelI9RoundLoopI13CfgPyrEuler29EEvi11EngineState6DynOut
64 32 0 0 _Z15dynamics_kernelI9RoundLoopI9CfgPyrRK4EEvi11EngineState6DynOut
- 0 0 0 _Z15forward_outputsI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E6FwdOut
- 0 0 0 _Z15forward_outputsI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E6FwdOut
- 0 0 0 _Z15forward_outputsI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E6FwdOut
- 0 0 0 _Z15forward_outputsI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E6FwdOut
- 0 0 12 _Z15make_constraintI11CfgEllEulerEviR4EnvSIT_E
- 0 0 12 _Z15make_constraintI11CfgPyrEulerEviR4EnvSIT_E
- 0 0 12 _Z15make_constraintI13CfgPyrEuler29EviR4EnvSIT_E
- 0 0 12 _Z15make_constraintI9CfgPyrRK4EviR4EnvSIT_E
- 0 0 0 _Z15make_constraintI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E
- 0 0 0 _Z15make_constraintI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E
- 0 0 0 _Z15make_constraintI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E
- 0 0 0 _Z15make_constraintI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E
- 0 0 0 _Z15mpr_penetrationPK10MprScratchPfS2_S2_S2_
- 0 0 0 _Z15update_gradientI11CfgEllEulerEfiR4EnvSIT_E
- 0 0 0 _Z15update_gradientI11CfgPyrEulerEfiR4EnvSIT_E
- 0 0 0 _Z15update_gradientI13CfgPyrEuler29EfiR4EnvSIT_E
- 0 0 0 _Z15update_gradientI9CfgPyrRK4EfiR4EnvSIT_E
- 0 0 0 _Z15update_gradientI9RoundLoopI11CfgEllEulerEEfiR4EnvSIT_E
- 0 0 0 _Z15update_gradientI9RoundLoopI11CfgPyrEulerEEfiR4EnvSIT_E
- 0 0 0 _Z15update_gradientI9RoundLoopI13CfgPyrEuler29EEfiR4EnvSIT_E
- 0 0 0 _Z15update_gradientI9RoundLoopI9CfgPyrRK4EEfiR4EnvSIT_E
- 0 0 0 _Z16forward_dynamicsI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E10SolverOpts6FwdOut
- 0 0 0 _Z16forward_dynamicsI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E10SolverOpts6FwdOut
- 0 0 0 _Z16forward_dynamicsI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E10SolverOpts6FwdOut
- 0 0 0 _Z16forward_dynamicsI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E10SolverOpts6FwdOut
- 0 0 0 _Z16inverse_dynamicsI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_EPf
- 0 0 0 _Z16inverse_dynamicsI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_EPf
- 0 0 0 _Z16inverse_dynamicsI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_EPf
- 0 0 0 _Z16inverse_dynamicsI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_EPf
- 0 40 84 _Z16physics_substepsI11CfgEllEulerEviR4EnvSIT_E10SolverOptsiPKii
- 0 40 84 _Z16physics_substepsI11CfgPyrEulerEviR4EnvSIT_E10SolverOptsiPKii
- 0 40 84 _Z16physics_substepsI13CfgPyrEuler29EviR4EnvSIT_E10SolverOptsiPKii
- 0 260 204 _Z16physics_substepsI9CfgPyrRK4EviR4EnvSIT_E10SolverOptsiPKii
- 0 0 0 _Z17constraint_updateI11CfgEllEulerEfiR4EnvSIT_E
- 0 0 0 _Z17constraint_updateI11CfgPyrEulerEfiR4EnvSIT_E
- 0 0 0 _Z17constraint_updateI13CfgPyrEuler29EfiR4EnvSIT_E
- 0 0 0 _Z17constraint_updateI9CfgPyrRK4EfiR4EnvSIT_E
- 0 0 0 _Z17constraint_updateI9RoundLoopI11CfgEllEulerEEfiR4EnvSIT_E
- 0 0 0 _Z17constraint_updateI9RoundLoopI11CfgPyrEulerEEfiR4EnvSIT_E
- 0 0 0 _Z17constraint_updateI9RoundLoopI13CfgPyrEuler29EEfiR4EnvSIT_E
- 0 0 0 _Z17constraint_updateI9RoundLoopI9CfgPyrRK4EEfiR4EnvSIT_E
- 0 0 0 _Z17convex_obb_filterI11CfgEllEulerEbiRK4EnvSIT_Ei
- 0 0 0 _Z17convex_obb_filterI11CfgPyrEulerEbiRK4EnvSIT_Ei
- 0 0 0 _Z17convex_obb_filterI13CfgPyrEuler29EbiRK4EnvSIT_Ei
- 0 0 0 _Z17convex_obb_filterI9CfgPyrRK4EbiRK4EnvSIT_Ei
- 0 0 0 _Z17convex_obb_filterI9RoundLoopI11CfgEllEulerEEbiRK4EnvSIT_Ei
- 0 0 0 _Z17convex_obb_filterI9RoundLoopI11CfgPyrEulerEEbiRK4EnvSIT_Ei
- 0 0 0 _Z17convex_obb_filterI9RoundLoopI13CfgPyrEuler29EEbiRK4EnvSIT_Ei
- 0 0 0 _Z17convex_obb_filterI9RoundLoopI9CfgPyrRK4EEbiRK4EnvSIT_Ei
- 0 0 0 _Z17finish_constraintI11CfgEllEulerEfiR4EnvSIT_E
- 0 0 0 _Z17finish_constraintI11CfgPyrEulerEfiR4EnvSIT_E
- 0 0 0 _Z17finish_constraintI13CfgPyrEuler29EfiR4EnvSIT_E
- 0 0 0 _Z17finish_constraintI9CfgPyrRK4EfiR4EnvSIT_E
- 0 0 0 _Z17finish_constraintI9RoundLoopI11CfgEllEulerEEfiR4EnvSIT_E
- 0 0 0 _Z17finish_constraintI9RoundLoopI11CfgPyrEulerEEfiR4EnvSIT_E
- 0 0 0 _Z17finish_constraintI9RoundLoopI13CfgPyrEuler29EEfiR4EnvSIT_E
- 0 0 0 _Z17finish_constraintI9RoundLoopI9CfgPyrRK4EEfiR4EnvSIT_E
56 0 0 0 _Z17load_state_kernel7DevTask11EngineStatePK4int4iPKiPfiiiiP4int2PiPh
- 0 0 0 _Z17make_hessian_wideI13CfgPyrEuler29EviR4EnvSIT_E
- 0 0 0 _Z17make_hessian_wideI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E
43 0 0 0 _Z17save_state_kernel7DevTask11EngineStatePKfP4int4iiiimlPK4int2
- 0 0 0 _Z17sphere_sphere_rawP6RawConfPKffS2_f
- 0 0 0 _Z17update_constraintI11CfgEllEulerEfiR4EnvSIT_EPf
- 0 0 0 _Z17update_constraintI11CfgPyrEulerEfiR4EnvSIT_EPf
- 0 0 0 _Z17update_constraintI13CfgPyrEuler29EfiR4EnvSIT_EPf
- 0 0 0 _Z17update_constraintI9CfgPyrRK4EfiR4EnvSIT_EPf
- 0 0 0 _Z17update_constraintI9RoundLoopI11CfgEllEulerEEfiR4EnvSIT_EPf
- 0 0 0 _Z17update_constraintI9RoundLoopI11CfgPyrEulerEEfiR4EnvSIT_EPf
- 0 0 0 _Z17update_constraintI9RoundLoopI13CfgPyrEuler29EEfiR4EnvSIT_EPf
- 0 0 0 _Z17update_constraintI9RoundLoopI9CfgPyrRK4EEfiR4EnvSIT_EPf
- 0 0 0 _Z18convex_hull_filterI11CfgEllEulerEbiRK4EnvSIT_Ei
- 0 0 0 _Z18convex_hull_filterI9RoundLoopI11CfgEllEulerEEbiRK4EnvSIT_Ei
- 0 0 0 _Z18make_hessian_splitI11CfgEllEulerEviR4EnvSIT_E
- 0 0 0 _Z18make_hessian_splitI11CfgPyrEulerEviR4EnvSIT_E
- 0 0 0 _Z18make_hessian_splitI9CfgPyrRK4EviR4EnvSIT_E
- 0 0 0 _Z18make_hessian_splitI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E
- 0 0 0 _Z18make_hessian_splitI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E
- 0 0 0 _Z18make_hessian_splitI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E
61 56 0 0 _Z19dataset_body_kernelI11CfgEllEulerEvi7DevTaskPKfPfS4_
61 56 0 0 _Z19dataset_body_kernelI11CfgPyrEulerEvi7DevTaskPKfPfS4_
63 56 0 0 _Z19dataset_body_kernelI13CfgPyrEuler29Evi7DevTaskPKfPfS4_
63 56 0 0 _Z19dataset_body_kernelI9CfgPyrRK4Evi7DevTaskPKfPfS4_
- 0 0 0 _Z4mulJI11CfgEllEulerEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulJI11CfgPyrEulerEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulJI13CfgPyrEuler29EviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulJI9CfgPyrRK4EviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulJI9RoundLoopI11CfgEllEulerEEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulJI9RoundLoopI11CfgPyrEulerEEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulJI9RoundLoopI13CfgPyrEuler29EEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulJI9RoundLoopI9CfgPyrRK4EEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulMI11CfgEllEulerEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulMI11CfgPyrEulerEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulMI13CfgPyrEuler29EviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulMI9CfgPyrRK4EviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulMI9RoundLoopI11CfgEllEulerEEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulMI9RoundLoopI11CfgPyrEulerEEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulMI9RoundLoopI13CfgPyrEuler29EEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z4mulMI9RoundLoopI9CfgPyrRK4EEviRK4EnvSIT_EPfPKf
- 0 0 0 _Z7com_posI11CfgEllEulerEviR4EnvSIT_E
- 0 0 0 _Z7com_posI11CfgPyrEulerEviR4EnvSIT_E
- 0 0 0 _Z7com_posI13CfgPyrEuler29EviR4EnvSIT_E
- 0 0 0 _Z7com_posI9CfgPyrRK4EviR4EnvSIT_E
- 0 0 0 _Z7com_posI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E
- 0 0 0 _Z7com_posI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E
- 0 0 0 _Z7com_posI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E
- 0 0 0 _Z7com_posI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E
- 0 32 4 _Z7forwardI11CfgEllEulerEviR4EnvSIT_E10SolverOpts
- 0 32 4 _Z7forwardI11CfgPyrEulerEviR4EnvSIT_E10SolverOpts
- 0 32 4 _Z7forwardI13CfgPyrEuler29EviR4EnvSIT_E10SolverOpts
- 0 36 28 _Z7forwardI9CfgPyrRK4EviR4EnvSIT_E10SolverOpts
- 0 0 0 _Z7forwardI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E10SolverOpts
- 0 0 0 _Z7forwardI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E10SolverOpts
- 0 0 0 _Z7forwardI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E10SolverOpts
- 0 0 0 _Z7forwardI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E10SolverOpts
- 0 0 0 _Z7ls_evalI11CfgEllEulerE7LSPointiRK4EnvSIT_EPKff
- 0 0 0 _Z7ls_evalI11CfgPyrEulerE7LSPointiRK4EnvSIT_EPKff
- 0 0 0 _Z7ls_evalI13CfgPyrEuler29E7LSPointiRK4EnvSIT_EPKff
- 0 0 0 _Z7ls_evalI9CfgPyrRK4E7LSPointiRK4EnvSIT_EPKff
- 0 0 0 _Z7ls_evalI9RoundLoopI11CfgEllEulerEE7LSPointiRK4EnvSIT_EPKff
- 0 0 0 _Z7ls_evalI9RoundLoopI11CfgPyrEulerEE7LSPointiRK4EnvSIT_EPKff
- 0 0 0 _Z7ls_evalI9RoundLoopI13CfgPyrEuler29EE7LSPointiRK4EnvSIT_EPKff
- 0 0 0 _Z7ls_evalI9RoundLoopI9CfgPyrRK4EE7LSPointiRK4EnvSIT_EPKff
- 0 28 156 _Z8rk4_stepI9CfgPyrRK4EviR4EnvSIT_E10SolverOpts
- 0 0 0 _Z9collisionI11CfgEllEulerEviR4EnvSIT_E
- 0 0 0 _Z9collisionI11CfgPyrEulerEviR4EnvSIT_E
- 0 0 0 _Z9collisionI13CfgPyrEuler29EviR4EnvSIT_E
- 0 0 0 _Z9collisionI9CfgPyrRK4EviR4EnvSIT_E
- 0 0 0 _Z9collisionI9RoundLoopI11CfgEllEulerEEviR4EnvSIT_E
- 0 0 0 _Z9collisionI9RoundLoopI11CfgPyrEulerEEviR4EnvSIT_E
- 0 0 0 _Z9collisionI9RoundLoopI13CfgPyrEuler29EEviR4EnvSIT_E
- 0 0 0 _Z9collisionI9RoundLoopI9CfgPyrRK4EEviR4EnvSIT_E
- 0 0 0 _Z9plane_boxP6RawConfPKfS2_S2_S2_S2_
- 0 0 0 _Z9reset_envI11CfgEllEulerEviRK7DevTaskR4EnvSIT_Eiif
- 0 0 0 _Z9reset_envI11CfgPyrEulerEviRK7DevTaskR4EnvSIT_Eiif
- 0 0 0 _Z9reset_envI13CfgPyrEuler29EviRK7DevTaskR4EnvSIT_Eiif
- 0 0 0 _Z9reset_envI9CfgPyrRK4EviRK7DevTaskR4EnvSIT_Eiif
30 0 0 0 dataset_kernel
24 0 0 0 fp32_peak_kernel
""",
    "locosim_configs31.cu": """
- 0 0 0 _ZN9locosim3110chol_solveILi31ELi32EEEvPAT0__fPf
- 0 0 0 _ZN9locosim3110convex_jobINS_12CfgPyrRK4_31EEEviRKNS_4EnvSIT_EERS4_iPf
- 0 0 0 _ZN9locosim3110convex_jobINS_13CfgPyrEuler31EEEviRKNS_4EnvSIT_EERS4_iPf
- 0 0 0 _ZN9locosim3110convex_jobINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRKNS_4EnvSIT_EERS6_iPf
- 0 0 0 _ZN9locosim3110convex_jobINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRKNS_4EnvSIT_EERS6_iPf
- 0 0 12 _ZN9locosim3110crb_factorINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EE
- 0 0 12 _ZN9locosim3110crb_factorINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3110crb_factorINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3110crb_factorINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3110euler_stepINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3110kinematicsINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3110kinematicsINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3110kinematicsINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3110kinematicsINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3110plane_meshEPNS_6RawConEfPKfS3_S3_S3_S3_if
- 0 0 0 _ZN9locosim3110sphere_boxEPNS_6RawConEfPKffS3_S3_S3_
72 56 0 0 _ZN9locosim3111body_kernelINS_12CfgPyrRK4_31EEEviNS_7DevTaskENS_11EngineStateEPKhS5_iimlPK4int2
71 56 0 0 _ZN9locosim3111body_kernelINS_13CfgPyrEuler31EEEviNS_7DevTaskENS_11EngineStateEPKhS5_iimlPK4int2
- 0 0 0 _ZN9locosim3111chol_factorILi31ELi32EEEviPAT0__f
- 0 0 0 _ZN9locosim3111dof_outputsINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3111dof_outputsINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3111line_searchINS_12CfgPyrRK4_31EEEfiRNS_4EnvSIT_EENS_10SolverOptsEfff
- 0 0 0 _ZN9locosim3111line_searchINS_13CfgPyrEuler31EEEfiRNS_4EnvSIT_EENS_10SolverOptsEfff
- 0 0 0 _ZN9locosim3111line_searchINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEfiRNS_4EnvSIT_EENS_10SolverOptsEfff
- 0 0 0 _ZN9locosim3111line_searchINS_9RoundLoopINS_13CfgPyrEuler31EEEEEfiRNS_4EnvSIT_EENS_10SolverOptsEfff
- 0 0 0 _ZN9locosim3111pair_narrowINS_12CfgPyrRK4_31EEEiiRNS_4EnvSIT_EEiPNS_6RawConEPiS8_Pf
- 0 0 0 _ZN9locosim3111pair_narrowINS_13CfgPyrEuler31EEEiiRNS_4EnvSIT_EEiPNS_6RawConEPiS8_Pf
- 0 0 0 _ZN9locosim3111pair_narrowINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEiiRNS_4EnvSIT_EEiPNS_6RawConEPiSA_Pf
- 0 0 0 _ZN9locosim3111pair_narrowINS_9RoundLoopINS_13CfgPyrEuler31EEEEEiiRNS_4EnvSIT_EEiPNS_6RawConEPiSA_Pf
14 0 0 0 _ZN9locosim3111rank_kernelEPKiPiii
128 688 312 400 _ZN9locosim3111step_kernelINS_12CfgPyrRK4_31EEEviNS_7DevTaskENS_10SolverOptsENS_11EngineStateEPKfPfS7_PhS7_iimliiPKhi
128 640 264 400 _ZN9locosim3111step_kernelINS_13CfgPyrEuler31EEEviNS_7DevTaskENS_10SolverOptsENS_11EngineStateEPKfPfS7_PhS7_iimliiPKhi
- 0 0 0 _ZN9locosim3112body_outputsINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EEPfS6_
- 0 0 0 _ZN9locosim3112body_outputsINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EEPfS6_
- 0 0 0 _ZN9locosim3112fill_contactINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EEiiifPKNS_6RawConE
- 0 0 0 _ZN9locosim3112fill_contactINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EEiiifPKNS_6RawConE
- 0 0 0 _ZN9locosim3112fill_contactINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EEiiifPKNS_6RawConE
- 0 0 0 _ZN9locosim3112fill_contactINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EEiiifPKNS_6RawConE
- 0 0 0 _ZN9locosim3112impedance_KBEPKfS1_fffPfS2_S2_
- 0 0 0 _ZN9locosim3112passive_biasINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3112passive_biasINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3112plane_sphereEPNS_6RawConEfPKfS3_S3_f
- 0 0 0 _ZN9locosim3113plane_capsuleEPNS_6RawConEfPKfS3_S3_S3_S3_
- 0 0 12 _ZN9locosim3113smooth_forcesINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EE
- 0 0 12 _ZN9locosim3113smooth_forcesINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3113smooth_forcesINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3113smooth_forcesINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3114contact_forcesINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EEPKii
- 0 0 0 _ZN9locosim3114contact_forcesINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EEPKii
- 0 0 0 _ZN9locosim3114contact_wrenchINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3114contact_wrenchINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3114convex_consumeINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EEiPKf
- 0 0 0 _ZN9locosim3114convex_consumeINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EEiPKf
- 0 0 0 _ZN9locosim3114convex_consumeINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EEiPKf
- 0 0 0 _ZN9locosim3114convex_consumeINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EEiPKf
- 0 0 0 _ZN9locosim3114dynamics_termsINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EENS_6DynOutE
- 0 0 0 _ZN9locosim3114dynamics_termsINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EENS_6DynOutE
128 320 0 0 _ZN9locosim3114forward_kernelINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviNS_11EngineStateENS_7DevTaskEPKiNS_10SolverOptsEPKfNS_6FwdOutE
128 320 0 0 _ZN9locosim3114forward_kernelINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviNS_11EngineStateENS_7DevTaskEPKiNS_10SolverOptsEPKfNS_6FwdOutE
- 0 0 36 _ZN9locosim3114fwd_constraintINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EENS_10SolverOptsE
- 0 0 32 _ZN9locosim3114fwd_constraintINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EENS_10SolverOptsE
- 0 0 0 _ZN9locosim3114fwd_constraintINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EENS_10SolverOptsE
- 0 0 0 _ZN9locosim3114fwd_constraintINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EENS_10SolverOptsE
- 0 0 0 _ZN9locosim3114init_workspaceINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3114init_workspaceINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3114init_workspaceINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3114init_workspaceINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EE
124 320 0 0 _ZN9locosim3114inverse_kernelINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviNS_11EngineStateENS_7DevTaskEPKiPKfS9_fPf
124 320 0 0 _ZN9locosim3114inverse_kernelINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviNS_11EngineStateENS_7DevTaskEPKiPKfS9_fPf
128 672 332 328 _ZN9locosim3114persist_kernelINS_12CfgPyrRK4_31EEEviNS_7DevTaskENS_10SolverOptsENS_11EngineStateEPKfPfS7_PhS7_iimliiPKhiNS_12PersistQueueE
128 624 268 328 _ZN9locosim3114persist_kernelINS_13CfgPyrEuler31EEEviNS_7DevTaskENS_10SolverOptsENS_11EngineStateEPKfPfS7_PhS7_iimliiPKhiNS_12PersistQueueE
- 0 0 0 _ZN9locosim3114plane_cylinderEPNS_6RawConEfPKfS3_S3_S3_S3_
- 0 0 0 _ZN9locosim3114sphere_capsuleEPNS_6RawConEfPKffS3_S3_S3_
128 688 284 364 _ZN9locosim3114substep_kernelINS_12CfgPyrRK4_31EEEviNS_7DevTaskENS_10SolverOptsENS_11EngineStateEPKfPfS7_PhS7_iimliiPKhiiiNS_10SplitStateE
128 624 228 344 _ZN9locosim3114substep_kernelINS_13CfgPyrEuler31EEEviNS_7DevTaskENS_10SolverOptsENS_11EngineStateEPKfPfS7_PhS7_iimliiPKhiiiNS_10SplitStateE
- 0 0 0 _ZN9locosim3115capsule_capsuleEPNS_6RawConEfPKfS3_S3_S3_S3_S3_
64 32 0 0 _ZN9locosim3115dynamics_kernelINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviNS_11EngineStateENS_6DynOutE
64 32 0 0 _ZN9locosim3115dynamics_kernelINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviNS_11EngineStateENS_6DynOutE
- 0 0 0 _ZN9locosim3115forward_outputsINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EENS_6FwdOutE
- 0 0 0 _ZN9locosim3115forward_outputsINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EENS_6FwdOutE
- 0 0 12 _ZN9locosim3115make_constraintINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EE
- 0 0 12 _ZN9locosim3115make_constraintINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3115make_constraintINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3115make_constraintINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3115mpr_penetrationEPKNS_10MprScratchEPfS3_S3_S3_
- 0 0 0 _ZN9locosim3115update_gradientINS_12CfgPyrRK4_31EEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3115update_gradientINS_13CfgPyrEuler31EEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3115update_gradientINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3115update_gradientINS_9RoundLoopINS_13CfgPyrEuler31EEEEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3116forward_dynamicsINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EENS_10SolverOptsENS_6FwdOutE
- 0 0 0 _ZN9locosim3116forward_dynamicsINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EENS_10SolverOptsENS_6FwdOutE
- 0 0 0 _ZN9locosim3116inverse_dynamicsINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EEPf
- 0 0 0 _ZN9locosim3116inverse_dynamicsINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EEPf
- 0 260 204 _ZN9locosim3116physics_substepsINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EENS_10SolverOptsEiPKii
- 0 40 84 _ZN9locosim3116physics_substepsINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EENS_10SolverOptsEiPKii
- 0 0 0 _ZN9locosim3117constraint_updateINS_12CfgPyrRK4_31EEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117constraint_updateINS_13CfgPyrEuler31EEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117constraint_updateINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117constraint_updateINS_9RoundLoopINS_13CfgPyrEuler31EEEEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117convex_obb_filterINS_12CfgPyrRK4_31EEEbiRKNS_4EnvSIT_EEi
- 0 0 0 _ZN9locosim3117convex_obb_filterINS_13CfgPyrEuler31EEEbiRKNS_4EnvSIT_EEi
- 0 0 0 _ZN9locosim3117convex_obb_filterINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEbiRKNS_4EnvSIT_EEi
- 0 0 0 _ZN9locosim3117convex_obb_filterINS_9RoundLoopINS_13CfgPyrEuler31EEEEEbiRKNS_4EnvSIT_EEi
- 0 0 0 _ZN9locosim3117finish_constraintINS_12CfgPyrRK4_31EEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117finish_constraintINS_13CfgPyrEuler31EEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117finish_constraintINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117finish_constraintINS_9RoundLoopINS_13CfgPyrEuler31EEEEEfiRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117make_hessian_wideINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117make_hessian_wideINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117make_hessian_wideINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117make_hessian_wideINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim3117sphere_sphere_rawEPNS_6RawConEfPKffS3_f
- 0 0 0 _ZN9locosim3117update_constraintINS_12CfgPyrRK4_31EEEfiRNS_4EnvSIT_EEPf
- 0 0 0 _ZN9locosim3117update_constraintINS_13CfgPyrEuler31EEEfiRNS_4EnvSIT_EEPf
- 0 0 0 _ZN9locosim3117update_constraintINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEfiRNS_4EnvSIT_EEPf
- 0 0 0 _ZN9locosim3117update_constraintINS_9RoundLoopINS_13CfgPyrEuler31EEEEEfiRNS_4EnvSIT_EEPf
63 56 0 0 _ZN9locosim3119dataset_body_kernelINS_12CfgPyrRK4_31EEEviNS_7DevTaskEPKfPfS5_
63 56 0 0 _ZN9locosim3119dataset_body_kernelINS_13CfgPyrEuler31EEEviNS_7DevTaskEPKfPfS5_
- 0 0 0 _ZN9locosim314mulJINS_12CfgPyrRK4_31EEEviRKNS_4EnvSIT_EEPfPKf
- 0 0 0 _ZN9locosim314mulJINS_13CfgPyrEuler31EEEviRKNS_4EnvSIT_EEPfPKf
- 0 0 0 _ZN9locosim314mulJINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRKNS_4EnvSIT_EEPfPKf
- 0 0 0 _ZN9locosim314mulJINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRKNS_4EnvSIT_EEPfPKf
- 0 0 0 _ZN9locosim314mulMINS_12CfgPyrRK4_31EEEviRKNS_4EnvSIT_EEPfPKf
- 0 0 0 _ZN9locosim314mulMINS_13CfgPyrEuler31EEEviRKNS_4EnvSIT_EEPfPKf
- 0 0 0 _ZN9locosim314mulMINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRKNS_4EnvSIT_EEPfPKf
- 0 0 0 _ZN9locosim314mulMINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRKNS_4EnvSIT_EEPfPKf
- 0 0 0 _ZN9locosim317com_posINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim317com_posINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim317com_posINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim317com_posINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EE
- 0 36 28 _ZN9locosim317forwardINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EENS_10SolverOptsE
- 0 32 4 _ZN9locosim317forwardINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EENS_10SolverOptsE
- 0 0 0 _ZN9locosim317forwardINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EENS_10SolverOptsE
- 0 0 0 _ZN9locosim317forwardINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EENS_10SolverOptsE
- 0 0 0 _ZN9locosim317ls_evalINS_12CfgPyrRK4_31EEENS_7LSPointEiRKNS_4EnvSIT_EEPKff
- 0 0 0 _ZN9locosim317ls_evalINS_13CfgPyrEuler31EEENS_7LSPointEiRKNS_4EnvSIT_EEPKff
- 0 0 0 _ZN9locosim317ls_evalINS_9RoundLoopINS_12CfgPyrRK4_31EEEEENS_7LSPointEiRKNS_4EnvSIT_EEPKff
- 0 0 0 _ZN9locosim317ls_evalINS_9RoundLoopINS_13CfgPyrEuler31EEEEENS_7LSPointEiRKNS_4EnvSIT_EEPKff
- 0 28 156 _ZN9locosim318rk4_stepINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EENS_10SolverOptsE
- 0 0 0 _ZN9locosim319collisionINS_12CfgPyrRK4_31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim319collisionINS_13CfgPyrEuler31EEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim319collisionINS_9RoundLoopINS_12CfgPyrRK4_31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim319collisionINS_9RoundLoopINS_13CfgPyrEuler31EEEEEviRNS_4EnvSIT_EE
- 0 0 0 _ZN9locosim319plane_boxEPNS_6RawConEfPKfS3_S3_S3_S3_
- 0 0 0 _ZN9locosim319reset_envINS_12CfgPyrRK4_31EEEviRKNS_7DevTaskERNS_4EnvSIT_EEiif
- 0 0 0 _ZN9locosim319reset_envINS_13CfgPyrEuler31EEEviRKNS_7DevTaskERNS_4EnvSIT_EEiif
""",
}


@pytest.mark.skipif(_nvcc_release() != "12.9", reason="the recorded figures are CUDA 12.9's")
def test_step_kernels_keep_the_parents_ptxas_figures(tmp_path):
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-prec-div=false",
             "-prec-sqrt=false", "-ftz=true", "-Xptxas", "-v", "-cubin"]
    procs = {}
    for unit in PARENT_FIGURES:
        src = os.path.join(ROOT, "loco_mujoco_b200", "csrc", unit)
        procs[unit] = subprocess.Popen([NVCC] + flags + ["-o", str(tmp_path / (unit + ".cubin")), src],
                                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    for unit, proc in procs.items():
        log, _ = proc.communicate()
        assert proc.returncode == 0, log[-3000:]
        now = ptxas_figures(log)
        want = {}
        for line in PARENT_FIGURES[unit].strip().splitlines():
            r, s, st, ld, name = line.split()
            want[name] = (None if r == "-" else int(r), int(s), int(st), int(ld))
        missing = sorted(set(want) - set(now))
        assert not missing, (unit, missing[:5])
        moved = {k: (want[k], now[k]) for k in want if now[k] != want[k]}
        assert not moved, (unit, moved)
        # the only new function is the writer itself, and it spills nothing
        new = {k: v for k, v in now.items() if k not in want}
        assert new and all("contact_list" in k for k in new), (unit, sorted(new))
        assert all(v[2] == 0 and v[3] == 0 for v in new.values()), new
