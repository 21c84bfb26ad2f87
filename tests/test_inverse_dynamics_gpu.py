"""Inverse dynamics on the GPU (include/locosim.h locosim_inverse / locosim_create_dataset_inverse; LocoEnv.inverse_dynamics /
create_dataset_inverse): parity with the fp64 reference (tests/inverse_ref.py) at the engine's own rollout states for every
kernel family and UnitreeA1 under position control, the call changes no bit of anything else on every launch path,
determinism, launch geometry and applied forces, non-finite inputs, the dataset bit for bit against pinned resets, CUDA
graphs, sharding and MixedBatch members."""
import os

import numpy as np
import pytest
import torch

import inverse_ref as ivr
from full_body import make_variant
from helpers import blobs, make_env
from position_mode import make_position

pytestmark = pytest.mark.gpu

# launch paths of UnitreeA1 (environment variables read when an engine is created, locosim.cu setup_cfg)
PATHS = {"fused": {"LOCOSIM_RESORT": "10"}, "substeps": {"LOCOSIM_RESORT": "2"},
         "persistent": {"LOCOSIM_RESORT": "2", "LOCOSIM_PERSIST": "1"}}
# one task per kernel family: CfgEllEuler (torque and position control), CfgPyrEuler, CfgPyrRK4, CfgPyrEuler29,
# CfgPyrRK4_31, CfgPyrEuler31
FAMILIES = ["UnitreeA1.simple", "UnitreeA1.simple+position", "Talos.walk", "HumanoidTorque.run", "UnitreeG1.walk",
            "Atlas.walk+arms", "Talos.walk+arms"]


@pytest.fixture(scope="module")
def ref():
    return ivr.load()


def _with_env(vars_, fn):
    old = {k: os.environ.get(k) for k in vars_}
    os.environ.update(vars_)
    try:
        return fn()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _make(task, path=None, **kw):
    if task.endswith("+position"):
        build = lambda: make_position(task[:-len("+position")], **kw)          # noqa: E731
    else:
        build = lambda: make_variant(task, **kw)                                # noqa: E731
    env = _with_env(PATHS[path] if path else {}, build)
    _with_env(PATHS[path] if path else {}, env._get_engine)
    return env


def _act(gen, n, nu):
    return (torch.rand((n, nu), generator=gen) * 2 - 1).cuda()


def _ctrl(spec, a):
    c = np.zeros(len(spec.act_idx))
    c[spec.act_idx] = a * spec.act_delta + spec.act_mean
    return c


@pytest.mark.parametrize("task", FAMILIES)
def test_matches_the_reference_at_rollout_states(ref, bundled_only, task):
    """States from the engine's own random-action rollouts (contacts active), evaluated in place: at the reference's forward
    qacc of random controls (the actuated dofs then come back as gear * force) and at random perturbations of it, within
    c 2^-23 S_d per dof; samples that fail it must be explained by the reference (tests/inverse_ref.py InverseSim.explained)
    and may be at most 5 % of the samples."""
    n, n_check = 256, 40
    env = _make(task, num_envs=n, seed=4)
    eng = env._get_engine()
    spec, m = env.task_spec(), env._model
    env.reset()
    gen = torch.Generator().manual_seed(3)
    for _ in range(6):
        env.step(_act(gen, n, m.nu))
    q, v, _ = (x.cpu().numpy() for x in eng.get_state())
    mb, tb = blobs(env)
    sim = ivr.InverseSim(ref, mb, tb, env._model_user_features[0], m.geom_type)
    rng = np.random.RandomState(9)
    rows = rng.choice(n, n_check, replace=False)
    qacc = np.zeros((2, n, m.nv), dtype=np.float32)
    act = {}
    for i in rows:
        a, f, _ = sim.forward(q[i].astype(np.float64), v[i].astype(np.float64), _ctrl(spec, rng.uniform(-1, 1, m.nu)))
        act[i] = f
        qacc[0, i] = a
        qacc[1, i] = a + rng.normal(0, 0.5, m.nv) * (1 + np.abs(a))
    total, ambiguous, constrained = 0, 0, 0
    for k in range(2):
        got = env.inverse_dynamics(torch.from_numpy(qacc[k]).cuda()).cpu().numpy()
        for i in rows:
            want = sim.at(q[i].astype(np.float64), v[i].astype(np.float64), qacc[k, i].astype(np.float64))
            total += 1
            constrained += int(np.abs(want["constraint"]).max() > 1.0)
            ok, ratio = ivr.within(got[i], want["qfrc"], want["scale"])
            if k == 0:
                actuated = act[i] != 0
                tol = ivr.C_TOL * ivr.EPS32 * want["scale"] + 1e-5 * np.abs(act[i]) + \
                    float(m.stat_meaninertia) * m.nv * 1e-5             # + the fp64 solver's own tolerance
                ok_act = bool(np.all(np.abs(got[i] - act[i])[actuated] <= tol[actuated]))
                ok = ok and ok_act
            if not ok:
                assert sim.explained(q[i].astype(np.float64), v[i].astype(np.float64), qacc[k, i].astype(np.float64), got[i],
                                     want["qfrc"]), (task, k, i, ratio)
                ambiguous += 1
    sim.close()
    print("%s: %d of %d samples outside the bound, each explained by the reference" % (task, ambiguous, total))
    assert ambiguous <= ivr.allowed(total), (task, ambiguous, total)
    assert constrained >= total // 4, (task, constrained, total)


@pytest.mark.parametrize("task,path", [("UnitreeA1.simple", "fused"), ("UnitreeA1.simple", "substeps"),
                                       ("UnitreeA1.simple", "persistent"), ("HumanoidTorque.run", None)])
def test_the_call_changes_nothing(bundled_only, task, path):
    """Twin engines, one calling inverse before every step: every output and every piece of engine state stays bit for
    bit the same"""
    n = 256
    a, b = _make(task, path, num_envs=n, seed=7), _make(task, path, num_envs=n, seed=7)
    for e in (a, b):
        e.body_state, e.contact_wrench, e.dof_outputs
    ea, eb = a._get_engine(), b._get_engine()
    assert torch.equal(a.reset(), b.reset())
    gen = torch.Generator().manual_seed(0)
    nu = a._model.nu
    for _ in range(6):
        qacc = torch.randn((n, a._model.nv), generator=gen).cuda()
        b.inverse_dynamics(qacc)
        act = _act(gen, n, nu)
        ra, rb = a.step(act), b.step(act)
        for x, y in zip(ra[:3], rb[:3]):
            assert torch.equal(x, y)
        assert torch.equal(ra[3]["next_obs"], rb[3]["next_obs"])
        for x, y in zip(ea.get_state(), eb.get_state()):
            assert torch.equal(x, y)
        assert torch.equal(ea.counters(), eb.counters()) and torch.equal(ea.cursor(), eb.cursor())
        for x, y in zip(ea.episode_stats(), eb.episode_stats()):
            assert torch.equal(x, y)
        for x, y in ((a.body_state, b.body_state), (a.next_body_state, b.next_body_state),
                     (a.contact_wrench, b.contact_wrench), (a.dof_outputs, b.dof_outputs)):
            assert torch.equal(x, y)


def test_determinism_geometry_and_applied_forces(bundled_only):
    """two calls give the same bits; an env's row is the same in engines of 1 and 512 envs at the same state; registered
    applied forces change no bit"""
    n = 512
    env = _make("UnitreeA1.simple", num_envs=n, seed=5)
    eng = env._get_engine()
    env.reset()
    gen = torch.Generator().manual_seed(1)
    for _ in range(4):
        env.step(_act(gen, n, 12))
    qacc = torch.randn((n, 18), generator=gen).cuda()
    r1, r2 = env.inverse_dynamics(qacc), env.inverse_dynamics(qacc)
    assert torch.equal(r1, r2) and bool(torch.isfinite(r1).all())
    env.xfrc_applied.normal_()
    env.qfrc_applied.normal_()
    assert torch.equal(env.inverse_dynamics(qacc), r1)
    q, v, w = eng.get_state()
    one = _make("UnitreeA1.simple", num_envs=1, seed=5)
    e1 = one._get_engine()
    for i in (0, 37, 511):
        e1.set_state(q[i:i + 1].contiguous(), v[i:i + 1].contiguous(), w[i:i + 1].contiguous())
        assert torch.equal(one.inverse_dynamics(qacc[i:i + 1].contiguous()), r1[i:i + 1])


def test_non_finite_inputs_give_zero_rows(bundled_only):
    n = 64
    env = _make("UnitreeA1.simple", num_envs=n, seed=2)
    eng = env._get_engine()
    env.reset()
    qacc = torch.randn((n, 18), device="cuda")
    base = env.inverse_dynamics(qacc)
    bad = qacc.clone()
    bad[3, 7] = float("nan")
    r = env.inverse_dynamics(bad)
    assert float(r[3].abs().max()) == 0.0
    keep = torch.arange(n, device="cuda") != 3
    assert torch.equal(r[keep], base[keep])
    # a non-finite stored state (a step would reset it: set_state keeps it)
    q, v, _ = eng.get_state()
    q[5, 3] = float("inf")
    v[9, 0] = float("nan")
    eng.set_state(q.contiguous(), v.contiguous())
    r = env.inverse_dynamics(qacc)
    assert float(r[5].abs().max()) == 0.0 and float(r[9].abs().max()) == 0.0 and bool(torch.isfinite(r).all())
    keep = (torch.arange(n, device="cuda") != 5) & (torch.arange(n, device="cuda") != 9)
    assert torch.equal(r[keep], base[keep])


@pytest.mark.parametrize("task,kw", [("UnitreeA1.simple", dict(setup_random_rot=True)), ("HumanoidTorque.run", {}),
                                     ("Atlas.walk+arms", {})])
def test_dataset_rows_equal_pinned_resets(bundled_only, task, kw):
    """Row r of create_dataset_inverse() equals, bit for bit, inverse on a twin engine reset onto the row's (traj, sample)
    with angle 0, at qacc = (v1 - v0) * inv_dt rebuilt in torch from the twin's velocities at sample and sample + 1"""
    env = _make(task, num_envs=8, seed=0, **kw)
    ds = env.create_dataset_inverse()
    m, spec = env._model, env.task_spec()
    n_traj, T = env.trajectories.number_of_trajectories, env.trajectories.trajectory_length
    per = T - 1
    assert ds.shape == (n_traj * per, m.nv) and len(env.create_dataset_device()["states"]) == len(ds)
    rows = torch.tensor([0, 1, per - 1, len(ds) - 1, len(ds) // 2, 7 * per + 3], dtype=torch.int64, device="cuda")
    rows = rows[rows < len(ds)]
    inv_dt = float(np.float32(1.0 / (float(np.float32(m.opt_timestep)) * spec.n_substeps)))
    twin = make_variant(task, num_envs=len(rows), **kw)
    eng = twin._get_engine()
    zero = torch.zeros(len(rows), device="cuda") if kw else None
    vel = []
    for c in (rows % per, rows % per + 1):
        eng.reset(traj_no=(rows // per).to(torch.int32).contiguous(), step_no=c.to(torch.int32).contiguous(), rot_angle=zero)
        vel.append(eng.get_state()[1].clone())
    eng.reset(traj_no=(rows // per).to(torch.int32).contiguous(), step_no=(rows % per).to(torch.int32).contiguous(),
              rot_angle=zero)
    qacc = (vel[1] - vel[0]) * torch.tensor(inv_dt, dtype=torch.float32, device="cuda")
    got = twin.inverse_dynamics(qacc.contiguous())
    assert torch.equal(got, ds[rows])
    assert bool(torch.isfinite(ds).all())


def test_captured_call_replays_on_new_inputs(bundled_only):
    n = 128
    env = _make("UnitreeA1.simple", num_envs=n, seed=8)
    eng = env._get_engine()
    env.reset()
    qacc = torch.randn((n, 18), device="cuda")
    out = torch.empty_like(qacc)
    eng.inverse(qacc, out)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            eng.inverse(qacc, out)
    gen = torch.Generator().manual_seed(3)
    for _ in range(3):
        env.step(_act(gen, n, 12))
        qacc.copy_(torch.randn((n, 18), generator=gen))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, env.inverse_dynamics(qacc))


def test_two_shards_equal_one_batch_and_mixed_batch_members(bundled_only):
    from loco_mujoco_b200.parallel import MixedBatch
    n = 64
    full = _make("UnitreeA1.simple", num_envs=n, seed=11)
    a = _make("UnitreeA1.simple", num_envs=n // 2, seed=11, env_id_offset=0)
    b = _make("UnitreeA1.simple", num_envs=n // 2, seed=11, env_id_offset=n // 2)
    assert torch.equal(full.reset(), torch.cat([a.reset(), b.reset()]))
    gen = torch.Generator().manual_seed(1)
    for _ in range(3):
        act = _act(gen, n, 12)
        full.step(act)
        a.step(act[:n // 2].contiguous())
        b.step(act[n // 2:].contiguous())
        qacc = torch.randn((n, 18), generator=gen).cuda()
        assert torch.equal(full.inverse_dynamics(qacc), torch.cat([a.inverse_dynamics(qacc[:n // 2].contiguous()),
                                                                   b.inverse_dynamics(qacc[n // 2:].contiguous())]))
    m = 48
    mb = MixedBatch([("Atlas.walk.real", m, {}), ("Talos.walk.real", m, {})], device="cuda:0", seed=3, debug=True)
    solo = [make_env("Atlas.walk", num_envs=m, seed=3, env_id_offset=0), make_env("Talos.walk", num_envs=m, seed=3, env_id_offset=m)]
    mb.reset()
    for e in solo:
        e.reset()
    acts = [_act(gen, m, e.action_dim) for e in mb.engines]
    mb.step(acts)
    for e, x in zip(solo, acts):
        e.step(x)
    torch.cuda.synchronize()
    for mem, s in zip(mb.envs, solo):
        qacc = torch.randn((m, s._model.nv), generator=gen).cuda()
        got = mem.inverse_dynamics(qacc)
        assert got.shape == (m, s._model.nv) and torch.equal(got, s.inverse_dynamics(qacc))


def test_each_env_uses_its_own_parameter_pool_row(ref, bundled_only):
    """tests/golden/dr_atlas_pool.npz (6 seeded randomised recompilations of Atlas, tools/make_dr_fixture.py) as the
    parameter pool: each env's row matches the fp64 reference built from its own pool row, and does not match one built
    from a deliberately wrong row"""
    from helpers import GOLDEN
    fx = np.load(os.path.join(GOLDEN, "dr_atlas_pool.npz"))
    pool, mints, mreals = fx["pool"], fx["model_ints"], fx["model_reals"]
    n = 48
    env = make_env("Atlas.walk", num_envs=n, seed=4)
    eng = env._get_engine()
    m, spec = env._model, env.task_spec()
    eng.set_param_pool(pool)
    rng = np.random.RandomState(0)
    tr = np.zeros(n, dtype=np.int32)
    st = rng.randint(0, env.trajectories.trajectory_length, n).astype(np.int32)
    eng.reset(traj_no=torch.tensor(tr, device=eng.device), step_no=torch.tensor(st, device=eng.device))
    for _ in range(3):
        eng.step(torch.tensor(rng.uniform(-1, 1, (n, eng.action_dim)), dtype=torch.float32, device=eng.device),
                 auto_reset=False)
    rows = eng.param_rows().cpu().numpy()
    assert len(set(rows.tolist())) > 1, "every env drew the same pool row"
    q, v, _ = (x.cpu().numpy().astype(np.float64) for x in eng.get_state())
    tb = spec.pack()
    # the deliberately wrong row of row r: the pool row whose parameters differ most from r's
    far = {r: int(np.argmax(np.abs(pool - pool[r]).max(axis=1))) for r in set(rows.tolist())}
    own = {r: ivr.InverseSim(ref, (mints, mreals[r]), tb, geom_type=m.geom_type) for r in set(rows.tolist())}
    wrong = {r: ivr.InverseSim(ref, (mints, mreals[far[r]]), tb, geom_type=m.geom_type) for r in set(rows.tolist())}
    qacc = np.zeros((n, m.nv), dtype=np.float32)
    for i in range(n):
        a, _, _ = own[rows[i]].forward(q[i], v[i], _ctrl(spec, rng.uniform(-1, 1, m.nu)))
        qacc[i] = a
    got = env.inverse_dynamics(torch.from_numpy(qacc).cuda()).cpu().numpy()
    explained, wrong_fails = 0, 0
    for i in range(n):
        want = own[rows[i]].at(q[i], v[i], qacc[i].astype(np.float64))
        ok, ratio = ivr.within(got[i], want["qfrc"], want["scale"])
        if not ok:
            assert own[rows[i]].explained(q[i], v[i], qacc[i].astype(np.float64), got[i], want["qfrc"]), (i, ratio)
            explained += 1
        other = wrong[rows[i]].at(q[i], v[i], qacc[i].astype(np.float64))
        bad, wrong_ratio = ivr.within(got[i], other["qfrc"], other["scale"])
        wrong_fails += int(not bad)
        assert wrong_ratio > ratio, (i, ratio, wrong_ratio)          # every env is closer to its own row than to the other
    for s in list(own.values()) + list(wrong.values()):
        s.close()
    print("pool rows: %d of %d envs outside the bound, each explained by the reference; %d of %d fail against a wrong row"
          % (explained, n, wrong_fails, n))
    assert explained <= ivr.allowed(n), (explained, n)
    assert wrong_fails >= n - n // 16, (wrong_fails, n)
