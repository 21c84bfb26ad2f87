"""Forward dynamics under an action on the GPU (include/locosim.h locosim_forward; LocoEnv.forward_dynamics): parity with the
fp64 reference (tests/forward_ref.py) at the engine's own rollout states for every kernel family, pool rows and carried
weights, the forward / inverse round trip with registered applied forces, identities against dynamics_terms, the call
changes nothing, non-finite rows, output subsets, CUDA graphs, sharding and MixedBatch members."""
import os

import numpy as np
import pytest
import torch

import forward_ref as fwr
import inverse_ref as ivr
from full_body import make_variant
from helpers import blobs, make_env
from position_mode import make_position

pytestmark = pytest.mark.gpu

G = 9.81
ALL = dict(dof=True, body_acc=True, cfrc_int=True, cfrc_ext=True)
# one task per kernel family: CfgEllEuler (torque and position control), CfgPyrEuler, CfgPyrRK4, CfgPyrEuler29,
# CfgPyrRK4_31, CfgPyrEuler31
FAMILIES = ["UnitreeA1.simple", "UnitreeA1.simple+position", "Talos.walk", "HumanoidTorque.run", "UnitreeG1.walk",
            "Atlas.walk+arms", "Talos.walk+arms"]


@pytest.fixture(scope="module")
def ref():
    return fwr.load()


def _make(task, **kw):
    if task.endswith("+position"):
        env = make_position(task[:-len("+position")], **kw)
    else:
        env = make_variant(task, **kw)
    env._get_engine()
    return env


def _act(gen, n, nu):
    return (torch.rand((n, nu), generator=gen) * 2 - 1).cuda()


def _ctrl(spec, a):
    c = np.zeros(len(spec.act_idx))
    c[spec.act_idx] = a * spec.act_delta + spec.act_mean
    return c


def _rollout(env, n, steps, seed):
    env.reset()
    gen = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        env.step(_act(gen, n, env._model.nu))
    return gen


def _np(out):
    return {k: x.cpu().numpy() for k, x in out.items()}


def _check_rows(env, ref, rows, got, action, xfrc=None, qfrc=None, model_of=None):
    """each env of `rows` against the fp64 reference of its model (model_of(i): index into env._models, default 0) at its
    stored state; a sample outside forward_ref.REL must be within 10x the reference's own jump: (samples, explained)"""
    eng = env._get_engine()
    spec = env.task_spec()
    q, v, _ = (x.cpu().numpy().astype(np.float64) for x in eng.get_state())
    sims, invs, explained = {}, {}, 0
    for i in rows:
        k = 0 if model_of is None else int(model_of(i))
        if k not in sims:
            mb, tb = blobs(env, k)
            sims[k] = fwr.ForwardSim(ref, mb, tb, env._model_user_features[k])
            invs[k] = ivr.InverseSim(ref, mb, tb, env._model_user_features[k], env._models[k].geom_type)
        r = sims[k]
        ctrl = _ctrl(spec, action[i].astype(np.float64))
        want = r.forward(q[i], v[i], ctrl, xfrc=None if xfrc is None else xfrc[i].astype(np.float64),
                         qfrc=None if qfrc is None else qfrc[i].astype(np.float64))
        ok = all(fwr.within(got[k2][i], want[k2], k2)[0] for k2 in fwr.OUTPUTS)
        if not ok and invs[k].mpr_contact(q[i], v[i]):
            # fp32 and fp64 MPR each stop at MPR's tolerance, on deep or near-tied portals on different faces
            explained += 1
            continue
        if not ok:
            gap = r.sensitivity(q[i], v[i], ctrl, want)
            for k2 in fwr.OUTPUTS:
                assert fwr.within(got[k2][i], want[k2], k2, gap[k2])[0], (k2, i, fwr.within(got[k2][i], want[k2], k2))
            explained += 1
    for r in list(sims.values()) + list(invs.values()):
        r.close()
    return len(rows), explained


@pytest.mark.parametrize("task", FAMILIES)
def test_matches_the_reference_at_rollout_states(ref, bundled_only, task):
    """80 envs at the engine's own random-action rollout states (contacts active) under new random actions, against the
    fp64 reference; samples outside the bound must be explained by the reference's own jump there, at most 5 %"""
    n = 256
    env = _make(task, num_envs=n, seed=4)
    gen = _rollout(env, n, 6, 3)
    action = _act(gen, n, env._model.nu)
    got = _np(env.forward_dynamics(action, **ALL))
    rows = np.random.RandomState(9).choice(n, 80, replace=False)
    total, explained = _check_rows(env, ref, rows, got, action.cpu().numpy())
    print("%s: %d of %d samples outside the bound, each explained by the reference" % (task, explained, total))
    assert explained <= int(0.05 * total), (task, explained, total)
    assert int((np.abs(got["cfrc_ext"][rows]).max(axis=(1, 2)) > 1.0).sum()) >= total // 4


@pytest.mark.parametrize("task", ["Atlas.carry", "UnitreeH1.carry"])
def test_carried_weights_and_pool_rows(ref, bundled_only, task):
    """every env follows its own pool row: the carried weight's model"""
    n = 64
    env = _make(task, num_envs=n, seed=6)
    gen = _rollout(env, n, 3, 5)
    rows = env._get_engine().param_rows().cpu().numpy()
    assert len(set(rows.tolist())) > 1
    action = _act(gen, n, env._model.nu)
    got = _np(env.forward_dynamics(action, **ALL))
    total, explained = _check_rows(env, ref, range(0, n, 2), got, action.cpu().numpy(), model_of=lambda i: rows[i])
    assert explained <= max(1, int(0.05 * total)), (task, explained, total)


def test_each_env_uses_its_own_parameter_pool_row(ref, bundled_only):
    from helpers import GOLDEN
    import dynamics_terms_ref as dtr
    fx = np.load(os.path.join(GOLDEN, "dr_atlas_pool.npz"))
    pool = fx["pool"]
    n = 48
    env = make_env("Atlas.walk", num_envs=n, seed=4)
    eng = env._get_engine()
    eng.set_param_pool(pool)
    gen = _rollout(env, n, 3, 0)
    rows = eng.param_rows().cpu().numpy()
    assert len(set(rows.tolist())) > 1
    env._models = [dtr.model_with_pool_row(env._model, pool[r]) for r in range(len(pool))]
    env._model_user_features = [()] * len(pool)
    action = _act(gen, n, env._model.nu)
    got = _np(env.forward_dynamics(action, **ALL))
    total, explained = _check_rows(env, ref, range(n), got, action.cpu().numpy(), model_of=lambda i: rows[i])
    assert explained <= max(1, int(0.05 * total)), (explained, total)


# ---------------------------------------------------------------------------------------------------------------------
# identities against the engine's other queries
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["UnitreeA1.simple", "HumanoidTorque.run", "Atlas.walk+arms"])
def test_forward_then_inverse_with_applied_forces(ref, bundled_only, task):
    """mjENBL_FWDINV at the engine's rollout states with registered applied forces: inverse_dynamics(qacc) =
    qfrc_actuator + qfrc_applied + J_xipos^T xfrc_applied up to the solver's convergence; and M qacc + bias - passive =
    qfrc_actuator + qfrc_constraint + the applied forces (dynamics_terms)"""
    n = 128
    env = _make(task, num_envs=n, seed=2)
    m = env._model
    gen = _rollout(env, n, 5, 1)
    env.xfrc_applied.copy_(torch.randn((n, m.nbody, 6), generator=gen).cuda() * 5)
    env.xfrc_applied[:, 0] = 0
    env.qfrc_applied.copy_(torch.randn((n, m.nv), generator=gen).cuda() * 5)
    action = _act(gen, n, m.nu)
    out = env.forward_dynamics(action)
    dof = out["dof"]
    qacc = dof[..., 2].contiguous()
    inv = env.inverse_dynamics(qacc)
    terms = env.dynamics_terms(body_jacobian=True)
    # J_xipos^T xfrc: the wrench at xipos moved to xpos, through the Jacobian at xpos
    q = env._get_engine().get_state()[0].cpu().numpy().astype(np.float64)
    mb, tb = blobs(env)
    r = fwr.ForwardSim(ref, mb, tb, env._model_user_features[0])
    xf = env.xfrc_applied.cpu().numpy().astype(np.float64)
    jac = terms["body_jacobian"].cpu().numpy().astype(np.float64)
    gen_x = np.zeros((n, m.nv))
    for i in range(n):
        xipos = r.forward(q[i], np.zeros(m.nv))["xipos"]
        xpos, _, _ = r.kin(q[i])
        for b in range(1, m.nbody):
            F, T = xf[i, b, :3], xf[i, b, 3:] + np.cross(xipos[b] - xpos[b], xf[i, b, :3])
            gen_x[i] += jac[i, b, 3:].T @ F + jac[i, b, :3].T @ T
    r.close()
    applied = env.qfrc_applied.cpu().numpy() + gen_x
    act = dof[..., 0].cpu().numpy()
    scale = 1.0 / (float(m.stat_meaninertia) * m.nv)
    res = inv.cpu().numpy() - act - applied
    ok = np.linalg.norm(res, axis=1) * scale < 1e-3
    assert ok.mean() >= 0.95, (task, np.sort(np.linalg.norm(res, axis=1) * scale)[-5:])
    M, bias, passive = (terms[k].cpu().numpy() for k in ("mass_matrix", "bias", "passive"))
    lhs = np.einsum("nij,nj->ni", M, qacc.cpu().numpy()) + bias - passive
    rhs = act + dof[..., 1].cpu().numpy() + applied
    ok = np.linalg.norm(lhs - rhs, axis=1) * scale < 1e-3                  # (an env that hit the iteration cap is not)
    assert ok.mean() >= 0.95, (task, np.sort(np.linalg.norm(lhs - rhs, axis=1) * scale)[-5:])


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "Talos.walk", "HumanoidTorque.run"])
def test_at_rest_accelerations_follow_the_jacobians(bundled_only, task):
    """At rollout states with qvel set to 0 (feet on the ground): body_acc = body_jacobian @ qacc - (0, g), and over the
    whole robot sum of cfrc_ext + M_total g = M_total jac_com @ qacc (dynamics_terms), plus the force the root's joints
    carry, cfrc_int[1] (friction loss and armature of the root slides: UnitreeA1's are 0.2 N each)"""
    n = 64
    env = _make(task, num_envs=n, seed=3)
    eng = env._get_engine()
    _rollout(env, n, 3, 2)
    q, v, w = eng.get_state()
    eng.set_state(q.contiguous(), torch.zeros_like(v), w.contiguous())
    gen = torch.Generator().manual_seed(5)
    out = env.forward_dynamics(_act(gen, n, env._model.nu), **ALL)
    terms = env.dynamics_terms(com=True, body_jacobian=True, com_jacobian=True)
    qacc = out["dof"][..., 2].double()
    acc = torch.einsum("nbrd,nd->nbr", terms["body_jacobian"].double(), qacc)
    acc[..., 5] += G
    acc[:, 0] = torch.tensor([0, 0, 0, 0, 0, G], dtype=torch.float64, device=acc.device)
    scale = acc.abs().amax(dim=(1, 2), keepdim=True).clamp(min=1.0)
    assert bool(((out["body_acc"].double() - acc).abs() <= 1e-3 * scale).all()), (task, (out["body_acc"].double() - acc).abs().max())
    mass = terms["com"][:, 3].double()
    lhs = out["cfrc_ext"][..., :3].double().sum(dim=1) + out["cfrc_int"][:, 1, :3].double()
    lhs[:, 2] -= mass * G
    rhs = mass[:, None] * torch.einsum("ncd,nd->nc", terms["com_jacobian"].double(), qacc)
    assert bool(((lhs - rhs).abs() <= 1e-3 * (mass * G)[:, None]).all()), (task, (lhs - rhs).abs().max())
    assert float(out["cfrc_ext"].abs().max()) > 0.0


# ---------------------------------------------------------------------------------------------------------------------
# call rules
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task,path", [("UnitreeA1.simple", None), ("UnitreeA1.simple", "fused"), ("HumanoidTorque.run", None)])
def test_the_call_changes_nothing(bundled_only, task, path):
    """Twin engines, one calling forward_dynamics before every step: every output and every piece of engine state stays
    bit for bit the same, the dof outputs (and their actuator scratch) included"""
    n = 256
    old = os.environ.get("LOCOSIM_RESORT")
    if path == "fused":
        os.environ["LOCOSIM_RESORT"] = "10"
    try:
        a, b = _make(task, num_envs=n, seed=7), _make(task, num_envs=n, seed=7)
    finally:
        if path == "fused":
            if old is None:
                os.environ.pop("LOCOSIM_RESORT", None)
            else:
                os.environ["LOCOSIM_RESORT"] = old
    for e in (a, b):
        e.body_state, e.contact_wrench, e.dof_outputs, e.xfrc_applied
    ea, eb = a._get_engine(), b._get_engine()
    assert torch.equal(a.reset(), b.reset())
    gen = torch.Generator().manual_seed(0)
    nu = a._model.nu
    for _ in range(6):
        b.forward_dynamics(_act(gen, n, nu), **ALL)
        act = _act(gen, n, nu)
        ra, rb = a.step(act), b.step(act)
        for x, y in zip(ra[:3], rb[:3]):
            assert torch.equal(x, y)
        for x, y in zip(ea.get_state(), eb.get_state()):
            assert torch.equal(x, y)
        assert torch.equal(ea.counters(), eb.counters()) and torch.equal(ea.cursor(), eb.cursor())
        for x, y in zip(ea.episode_stats(), eb.episode_stats()):
            assert torch.equal(x, y)
        for x, y in ((a.body_state, b.body_state), (a.next_body_state, b.next_body_state),
                     (a.contact_wrench, b.contact_wrench), (a.dof_outputs, b.dof_outputs)):
            assert torch.equal(x, y)


def test_subsets_non_finite_rows_and_geometry(bundled_only):
    """any subset of outputs gives the bits of all four; a non-finite state or action gives zero rows and leaves the other
    rows' bits; an env's rows are the same in engines of 1 and 512 envs"""
    n = 512
    env = _make("UnitreeA1.simple", num_envs=n, seed=5)
    eng = env._get_engine()
    gen = _rollout(env, n, 4, 1)
    action = _act(gen, n, 12)
    full = {k: x.clone() for k, x in env.forward_dynamics(action, **ALL).items()}
    assert all(bool(torch.isfinite(x).all()) for x in full.values())
    for k in fwr.OUTPUTS:
        one = env.forward_dynamics(action, **{k2: k2 == k for k2 in fwr.OUTPUTS})
        assert list(one) == [k] and torch.equal(one[k], full[k])
    bad = action.clone()
    bad[3, 7] = float("nan")
    r = env.forward_dynamics(bad, **ALL)
    keep = torch.arange(n, device="cuda") != 3
    for k in fwr.OUTPUTS:
        assert float(r[k][3].abs().max()) == 0.0 and torch.equal(r[k][keep], full[k][keep])
    q, v, w = eng.get_state()
    one = _make("UnitreeA1.simple", num_envs=1, seed=5)
    e1 = one._get_engine()
    for i in (0, 37, 511):
        e1.set_state(q[i:i + 1].contiguous(), v[i:i + 1].contiguous(), w[i:i + 1].contiguous())
        r1 = one.forward_dynamics(action[i:i + 1].contiguous(), **ALL)
        for k in fwr.OUTPUTS:
            assert torch.equal(r1[k], full[k][i:i + 1]), (i, k)
    q = q.clone()
    v = v.clone()
    q[5, 3] = float("inf")
    v[9, 0] = float("nan")
    eng.set_state(q.contiguous(), v.contiguous(), w.contiguous())
    r = env.forward_dynamics(action, **ALL)
    keep = (torch.arange(n, device="cuda") != 5) & (torch.arange(n, device="cuda") != 9)
    for k in fwr.OUTPUTS:
        assert float(r[k][5].abs().max()) == 0.0 and float(r[k][9].abs().max()) == 0.0
        assert torch.equal(r[k][keep], full[k][keep])


def test_captured_call_replays_on_new_actions_and_states(bundled_only):
    n = 128
    env = _make("UnitreeA1.simple", num_envs=n, seed=8)
    env.reset()
    action = torch.zeros((n, 12), device="cuda")
    out = env.forward_dynamics(action, **ALL)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            env.forward_dynamics(action, out=out, **ALL)
    gen = torch.Generator().manual_seed(3)
    for _ in range(3):
        env.step(_act(gen, n, 12))
        action.copy_(_act(gen, n, 12))
        graph.replay()
        torch.cuda.synchronize()
        want = env.forward_dynamics(action, **ALL)
        for k in fwr.OUTPUTS:
            assert torch.equal(out[k], want[k]), k


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
        x = _act(gen, n, 12)
        f = full.forward_dynamics(x, **ALL)
        fa, fb = a.forward_dynamics(x[:n // 2].contiguous(), **ALL), b.forward_dynamics(x[n // 2:].contiguous(), **ALL)
        for k in fwr.OUTPUTS:
            assert torch.equal(f[k], torch.cat([fa[k], fb[k]])), k
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
        x = _act(gen, m, s._model.nu)
        got, want = mem.forward_dynamics(x, **ALL), s.forward_dynamics(x, **ALL)
        for k in fwr.OUTPUTS:
            assert got[k].shape == want[k].shape and torch.equal(got[k], want[k]), k
