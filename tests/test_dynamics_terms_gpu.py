"""Dynamics terms on the GPU (include/locosim.h locosim_dynamics_terms; LocoEnv.dynamics_terms): parity with the fp64 reference
(tests/dynamics_terms_ref.py) at the engine's own rollout states for every kernel family and UnitreeA1 under position
control, parameter-pool rows and carried weights, identities against the engine's other outputs (body_state,
inverse_dynamics), the call changes no bit of anything else, non-finite states, CUDA graphs, sharding and MixedBatch
members."""
import os

import numpy as np
import pytest
import torch

import dynamics_terms_ref as dtr
from full_body import make_variant
from helpers import make_env
from position_mode import make_position

pytestmark = pytest.mark.gpu

# one task per kernel family: CfgEllEuler (torque and position control), CfgPyrEuler, CfgPyrRK4, CfgPyrEuler29,
# CfgPyrRK4_31, CfgPyrEuler31
FAMILIES = ["UnitreeA1.simple", "UnitreeA1.simple+position", "Talos.walk", "HumanoidTorque.run", "UnitreeG1.walk",
            "Atlas.walk+arms", "Talos.walk+arms"]
ALL = dict(mass_matrix=True, bias=True, passive=True, com=True, body_jacobian=True, com_jacobian=True)
KEYS = {"mass_matrix": "M", "bias": "bias", "passive": "passive", "com": "com", "body_jacobian": "jac",
        "com_jacobian": "jac_com"}


@pytest.fixture(scope="module")
def ref():
    return dtr.load()


def _make(task, **kw):
    if task.endswith("+position"):
        return make_position(task[:-len("+position")], **kw)
    return make_variant(task, **kw)


def _act(gen, n, nu):
    return (torch.rand((n, nu), generator=gen) * 2 - 1).cuda()


def _rollout(env, n, steps, seed):
    env.reset()
    gen = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        env.step(_act(gen, n, env._model.nu))


def _row(terms, i):
    """env i's terms as numpy arrays, keyed as dynamics_terms_ref"""
    return {KEYS[k]: x[i].cpu().numpy() for k, x in terms.items()}


@pytest.mark.parametrize("task", FAMILIES)
def test_matches_the_reference_at_rollout_states(ref, bundled_only, task):
    """States from the engine's own random-action rollouts (contacts active), 80 envs per family: every term within
    dynamics_terms_ref's fp32 error model at the stored state"""
    n, n_check = 256, 80
    env = _make(task, num_envs=n, seed=4)
    eng = env._get_engine()
    m = env._model
    _rollout(env, n, 6, 3)
    terms = env.dynamics_terms(**ALL)
    q, v, _ = (x.cpu().numpy().astype(np.float64) for x in eng.get_state())
    finite = np.flatnonzero(np.isfinite(q).all(1) & np.isfinite(v).all(1))
    rows = np.random.RandomState(9).choice(finite, n_check, replace=False)
    r = dtr.DynRef(ref, m)
    worst = {}
    for i in rows:
        for k, x in dtr.check(_row(terms, i), r.terms(q[i], v[i])).items():
            worst[k] = max(worst.get(k, 0.0), x)
    r.close()
    print("%s: largest error / bound per term over %d envs: %s" % (task, n_check,
                                                                   ", ".join("%s %.3g" % kv for kv in sorted(worst.items()))))


def test_each_env_uses_its_own_parameter_pool_row(ref, bundled_only):
    """tests/golden/dr_atlas_pool.npz (6 seeded randomised recompilations of Atlas) as the parameter pool: each env's terms
    match the reference of a model carrying its own pool row, and its total mass is that row's"""
    from helpers import GOLDEN
    fx = np.load(os.path.join(GOLDEN, "dr_atlas_pool.npz"))
    pool = fx["pool"]
    n = 48
    env = make_env("Atlas.walk", num_envs=n, seed=4)
    eng = env._get_engine()
    m = env._model
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
    terms = env.dynamics_terms(**ALL)
    refs = {r: dtr.DynRef(ref, dtr.model_with_pool_row(m, pool[r])) for r in set(rows.tolist())}
    masses = {r: float(np.sum(dtr.model_with_pool_row(m, pool[r]).body_mass)) for r in refs}
    assert len(set(masses.values())) > 1
    for i in range(n):
        got = _row(terms, i)
        dtr.check(got, refs[rows[i]].terms(q[i], v[i]))
        assert abs(got["com"][3] - masses[rows[i]]) <= 1e-6 * masses[rows[i]]
    for s in refs.values():
        s.close()


@pytest.mark.parametrize("task", ["Atlas.carry", "Talos.carry"])
def test_carry_tasks_follow_the_carried_weight(ref, bundled_only, task):
    """In a carry task every env's row follows its pool row, the carried weight's model: com[:, 3] is that model's total
    mass and every term matches that model's reference"""
    n = 64
    env = _make(task, num_envs=n, seed=6)
    eng = env._get_engine()
    _rollout(env, n, 3, 5)
    rows = eng.param_rows().cpu().numpy()
    assert len(set(rows.tolist())) > 1
    q, v, _ = (x.cpu().numpy().astype(np.float64) for x in eng.get_state())
    terms = env.dynamics_terms(**ALL)
    com = terms["com"].cpu().numpy()
    refs = {r: dtr.DynRef(ref, env._models[r]) for r in set(rows.tolist())}
    for i in range(n):
        mass = float(np.sum(env._models[rows[i]].body_mass))
        assert abs(com[i, 3] - mass) <= 1e-6 * mass, (i, com[i, 3], mass)
        if i % 4 == 0 and np.isfinite(q[i]).all() and np.isfinite(v[i]).all():
            dtr.check(_row(terms, i), refs[rows[i]].terms(q[i], v[i]))
    for s in refs.values():
        s.close()


# ---------------------------------------------------------------------------------------------------------------------
# identities against the engine's other outputs
# ---------------------------------------------------------------------------------------------------------------------
def _quat_rot(q, v):
    """rotate v [..., 3] by unit quaternions q [..., 4] (w x y z)"""
    w, u = q[..., :1], q[..., 1:]
    t = 2 * torch.cross(u, v, dim=-1)
    return v + w * t + torch.cross(u, t, dim=-1)


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "HumanoidTorque.run", "Atlas.walk+arms"])
def test_jacobians_give_the_body_and_com_velocities(bundled_only, task):
    """jac @ qvel = next_body_state[..., 7:13] and jac_com @ qvel = sum_b m_b v(xipos_b) / sum_b m_b from the body states,
    within fp32 rounding of the products summed (2^-23 C_TOL (1 + P) (|jac| |qvel|))"""
    n = 256
    env = _make(task, num_envs=n, seed=12)
    nb = env.next_body_state
    eng = env._get_engine()
    _rollout(env, n, 5, 2)
    terms = env.dynamics_terms(**ALL)
    _, v, _ = eng.get_state()
    ok = torch.isfinite(v).all(1)
    J, Jc = terms["body_jacobian"], terms["com_jacobian"]
    P = 1.0 + nb[..., :3].abs().amax((1, 2))[:, None, None]
    tol = dtr.C_TOL * dtr.EPS32 * P * ((J.abs() @ v.abs()[:, None, :, None])[..., 0] + 1e-3)
    got = (J @ v[:, None, :, None])[..., 0]
    err = (got - nb[..., 7:13]).abs()
    assert bool((err[ok] <= tol[ok]).all()), float((err / tol)[ok].max())
    m = env._model
    mass = torch.tensor(np.asarray(m.body_mass), dtype=torch.float32, device="cuda")
    ipos = torch.tensor(np.asarray(m.body_ipos).reshape(-1, 3), dtype=torch.float32, device="cuda")
    off = _quat_rot(nb[..., 3:7], ipos.expand(n, -1, -1))
    vi = nb[..., 10:13] + torch.cross(nb[..., 7:10], off, dim=-1)
    vcom = (mass[None, :, None] * vi).sum(1) / mass.sum()
    got = (Jc @ v[:, :, None])[..., 0]
    tol = dtr.C_TOL * dtr.EPS32 * P[:, :, 0] * ((Jc.abs() @ v.abs()[:, :, None])[..., 0] + 1e-3)
    err = (got - vcom).abs()
    assert bool((err[ok] <= tol[ok]).all()), float((err / tol)[ok].max())


@pytest.mark.parametrize("task", ["HumanoidTorque.run", "Atlas.walk+arms"])
def test_terms_sum_to_inverse_dynamics_without_constraints(ref, bundled_only, task):
    """M qacc + bias - passive = inverse_dynamics(qacc) where the state has no constraint row: reset-table states lifted
    2 m clear of the floor, hinges moved 0.02 rad inside their limits, and only envs whose state gives the fp64 reference
    no constraint row (HumanoidTorque has bone-bone contacts). (UnitreeA1 and Talos are left out: their dof_frictionloss
    rows are present at every state.) Within the reference's error scales of the three terms; at least 16 envs checked."""
    import ctypes
    n = 128
    env = _make(task, num_envs=n, seed=3)
    eng = env._get_engine()
    m = env._model
    assert not np.any(np.asarray(m.dof_frictionloss))
    env.reset()
    q, v, w = eng.get_state()
    axes = np.asarray(m.jnt_axis).reshape(-1, 3)
    zi = [j for j in range(3) if m.jnt_type[j] == m.jnt_type[0] and axes[j, 2] == 1.0]
    assert len(zi) == 1
    q = q.clone()
    q[:, zi[0]] += 2.0
    lim = np.asarray(m.jnt_limited).astype(bool)
    rng = torch.tensor(np.asarray(m.jnt_range), dtype=torch.float32, device="cuda")
    for j in np.flatnonzero(lim):
        q[:, j] = q[:, j].clamp(float(rng[j, 0]) + 0.02, float(rng[j, 1]) - 0.02)
    eng.set_state(q.contiguous(), v.contiguous(), w.contiguous())
    gen = torch.Generator().manual_seed(4)
    qacc = torch.randn((n, m.nv), generator=gen).cuda()
    terms = env.dynamics_terms()
    lhs = (terms["mass_matrix"] @ qacc[:, :, None])[..., 0] + terms["bias"] - terms["passive"]
    inv = env.inverse_dynamics(qacc)
    r = dtr.DynRef(ref, m)
    r.lib.ref_nefc.restype = ctypes.c_int
    r.lib.ref_nefc.argtypes = [ctypes.c_void_p]
    qn, vn, an = (x.cpu().numpy().astype(np.float64) for x in (q, v, qacc))
    lhs, inv = lhs.cpu().numpy(), inv.cpu().numpy()
    checked = 0
    for i in range(n):
        t = r.terms(qn[i], vn[i], jac=False)
        if r.lib.ref_nefc(r.sim) != 0:
            continue
        checked += 1
        scale = t["s_M"] @ np.abs(an[i]) + t["s_bias"] + t["s_passive"]
        ok, ratio = dtr.within(lhs[i], inv[i], scale)
        assert ok, (i, ratio)
    r.close()
    assert checked >= 16, (checked, n)


# ---------------------------------------------------------------------------------------------------------------------
# the call changes nothing; non-finite states; graphs; shards
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["UnitreeA1.simple", "HumanoidTorque.run"])
def test_the_call_changes_nothing(bundled_only, task):
    """Twin engines, one calling dynamics_terms (every output) before every step: every output and every piece of engine
    state stays bit for bit the same"""
    n = 256
    a, b = _make(task, num_envs=n, seed=7), _make(task, num_envs=n, seed=7)
    for e in (a, b):
        e.body_state, e.contact_wrench, e.dof_outputs
    ea, eb = a._get_engine(), b._get_engine()
    assert torch.equal(a.reset(), b.reset())
    gen = torch.Generator().manual_seed(0)
    nu = a._model.nu
    out = None
    for _ in range(6):
        q0 = [x.clone() for x in eb.get_state()]
        c0 = eb.counters().clone()
        out = b.dynamics_terms(**ALL, out=out)
        for x, y in zip(q0, eb.get_state()):
            assert torch.equal(x, y)
        assert torch.equal(c0, eb.counters())
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


def test_non_finite_state_gives_zero_rows_and_the_rest_is_unchanged(bundled_only):
    n = 64
    env = _make("UnitreeA1.simple", num_envs=n, seed=2)
    eng = env._get_engine()
    env.reset()
    base = {k: x.clone() for k, x in env.dynamics_terms(**ALL).items()}
    q, v, _ = eng.get_state()
    q[5, 3] = float("inf")
    v[9, 0] = float("nan")
    eng.set_state(q.contiguous(), v.contiguous())
    got = env.dynamics_terms(**ALL)
    keep = (torch.arange(n, device="cuda") != 5) & (torch.arange(n, device="cuda") != 9)
    for k, x in got.items():
        assert float(x[5].abs().max()) == 0.0 and float(x[9].abs().max()) == 0.0, k
        assert bool(torch.isfinite(x).all()) and torch.equal(x[keep], base[k][keep]), k


def test_determinism_geometry_and_what_is_asked_for(bundled_only):
    """two calls give the same bits; an env's rows are the same in engines of 1 and 512 envs at the same state; asking for
    fewer terms gives the same bits of those terms and writes nothing else; body 0 is zeros"""
    n = 512
    env = _make("UnitreeA1.simple", num_envs=n, seed=5)
    eng = env._get_engine()
    _rollout(env, n, 4, 1)
    r1 = {k: x.clone() for k, x in env.dynamics_terms(**ALL).items()}
    r2 = env.dynamics_terms(**ALL)
    assert all(torch.equal(r1[k], r2[k]) for k in r1)
    assert float(r1["body_jacobian"][:, 0].abs().max()) == 0.0
    for k in ALL:
        only = {kk: kk == k for kk in ALL}
        got = env.dynamics_terms(**only)
        assert list(got) == [k] and torch.equal(got[k], r1[k])
    sentinel = {k: torch.full_like(x, 7.0) for k, x in r1.items()}
    out = env.dynamics_terms(mass_matrix=False, bias=True, passive=False, com=False, out=sentinel)
    assert out is sentinel and torch.equal(out["bias"], r1["bias"])
    assert all(bool((out[k] == 7.0).all()) for k in out if k != "bias")
    q, v, w = eng.get_state()
    one = _make("UnitreeA1.simple", num_envs=1, seed=5)
    e1 = one._get_engine()
    for i in (0, 37, 511):
        e1.set_state(q[i:i + 1].contiguous(), v[i:i + 1].contiguous(), w[i:i + 1].contiguous())
        got = one.dynamics_terms(**ALL)
        assert all(torch.equal(got[k], r1[k][i:i + 1]) for k in got)


def test_captured_call_replays_on_a_new_state(bundled_only):
    n = 128
    env = _make("UnitreeA1.simple", num_envs=n, seed=8)
    eng = env._get_engine()
    env.reset()
    out = env.dynamics_terms(**ALL)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            env.dynamics_terms(**ALL, out=out)
    gen = torch.Generator().manual_seed(3)
    for _ in range(3):
        env.step(_act(gen, n, 12))
        graph.replay()
        torch.cuda.synchronize()
        eager = env.dynamics_terms(**ALL)
        assert all(torch.equal(out[k], eager[k]) for k in out)


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
        fa, fb, ff = a.dynamics_terms(**ALL), b.dynamics_terms(**ALL), full.dynamics_terms(**ALL)
        for k in ff:
            assert torch.equal(ff[k], torch.cat([fa[k], fb[k]])), k
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
        got, want = mem.dynamics_terms(**ALL), s.dynamics_terms(**ALL)
        assert got["mass_matrix"].shape == (m, s._model.nv, s._model.nv)
        assert all(torch.equal(got[k], want[k]) for k in want)
