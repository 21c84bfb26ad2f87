"""Applied forces on the GPU (include/locosim.h locosim_set_applied_forces; LocoEnv.xfrc_applied / qfrc_applied): off is
off, parity with the fp64 reference (tests/csrc/applied_forces_ref.c) for every kernel family, the three launch paths bit for
bit, momentum, resets, CUDA graphs, sharding."""
import os

import numpy as np
import pytest
import torch

import applied_forces_ref
from full_body import make_variant
from helpers import blobs, make_env

pytestmark = pytest.mark.gpu

# launch paths of UnitreeA1 (environment variables read when an engine is created, include/locosim.h / locosim.cu)
PATHS = {"fused": {"LOCOSIM_RESORT": "10"}, "substeps": {"LOCOSIM_RESORT": "2"},
         "persistent": {"LOCOSIM_RESORT": "2", "LOCOSIM_PERSIST": "1"}}


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
    env = _with_env(PATHS[path] if path else {}, lambda: make_variant(task, **kw))
    _with_env(PATHS[path] if path else {}, env._get_engine)
    return env


@pytest.fixture(scope="module")
def ref():
    return applied_forces_ref.load()


def _random_forces(env, gen, frac=0.5):
    """wrenches on one random body of a random `frac` of the envs, random joint forces everywhere (on the device)"""
    n, nb, nv = env.num_envs, env._model.nbody, env._model.nv
    x = torch.zeros((n, nb, 6))
    hit = torch.rand(n, generator=gen) < frac
    body = torch.randint(1, nb, (n,), generator=gen)
    x[hit, body[hit]] = torch.randn((int(hit.sum()), 6), generator=gen) * torch.tensor([30., 30, 30, 3, 3, 3])
    return x.cuda(), (torch.randn((n, nv), generator=gen) * 2).cuda()


@pytest.mark.parametrize("task,path", [("UnitreeA1.simple", "fused"), ("UnitreeA1.simple", "substeps"),
                                       ("UnitreeA1.simple", "persistent"), ("HumanoidTorque.run", None),
                                       ("Atlas.walk+arms", None)])
def test_zero_buffers_change_no_bit(bundled_only, task, path):
    """512 envs: an engine with zero buffers registered steps bit for bit like one without (fused kernel, sub-step launches,
    persistent kernel, an RK4 configuration, a 31-dof configuration), auto-resets included."""
    n = 512
    a, b = _make(task, path, num_envs=n, seed=7), _make(task, path, num_envs=n, seed=7)
    b.xfrc_applied, b.qfrc_applied                     # allocated zeroed and registered
    assert torch.equal(a.reset(), b.reset())
    gen = torch.Generator().manual_seed(0)
    nu = a.info.action_space.shape[0]
    for _ in range(6):
        act = (torch.rand((n, nu), generator=gen) * 2 - 1).cuda()
        ra, rb = a.step(act), b.step(act)
        for x, y in zip(ra[:3], rb[:3]):
            assert torch.equal(x, y)
        assert torch.equal(ra[3]["next_obs"], rb[3]["next_obs"])
    for x, y in zip(a._get_engine().get_state(), b._get_engine().get_state()):
        assert torch.equal(x, y)
    assert float(b.xfrc_applied.abs().max()) == 0 and float(b.qfrc_applied.abs().max()) == 0


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "HumanoidTorque.run", "Atlas.walk", "Talos.walk", "UnitreeG1.walk",
                                  "Atlas.walk+arms"])
def test_forces_match_the_reference(ref, bundled_only, task):
    """random wrenches on random bodies plus random joint forces, three control steps from pinned resets, against the fp64
    reference with the tolerance of test_gpu_parity (2e-3 (k + 1)); an env whose step crosses a contact switch may leave the
    fp64 branch (at most 1 in 8)."""
    n = 48
    env = make_variant(task, num_envs=n, seed=5)
    eng = env._get_engine()
    mb, tb = blobs(env)
    rng = np.random.RandomState(0)
    tr = rng.randint(0, env.trajectories.number_of_trajectories, n).astype(np.int32)
    st = rng.randint(0, env.trajectories.trajectory_length - 5, n).astype(np.int32)
    eng.reset(traj_no=torch.tensor(tr, device=eng.device), step_no=torch.tensor(st, device=eng.device))
    sims = [applied_forces_ref.AppliedSim(ref, mb, tb, env._model_user_features[0]) for _ in range(n)]
    for i, s in enumerate(sims):
        s.reset_to(tr[i], st[i])
    gen = torch.Generator().manual_seed(1)
    alive, off = np.ones(n, dtype=bool), 0
    for k in range(3):
        x, q = _random_forces(env, gen)
        env.xfrc_applied.copy_(x)
        env.qfrc_applied.copy_(q)
        act = rng.uniform(-1, 1, (n, eng.action_dim)).astype(np.float32)
        eng.step(torch.tensor(act, device=eng.device), auto_reset=False)
        qg, vg, _ = (t.cpu().numpy() for t in eng.get_state())
        xh, qh = x.cpu().numpy().astype(np.float64), q.cpu().numpy().astype(np.float64)
        for i in range(n):
            if not alive[i]:
                continue
            qo, vo = sims[i].env_step(act[i], xfrc=xh[i], qfrc=qh[i])
            tol = 2e-3 * (k + 1)
            if not (np.allclose(qg[i], qo, rtol=tol, atol=tol) and np.allclose(vg[i], vo, rtol=tol, atol=tol)):
                off += 1
                alive[i] = False
    for s in sims:
        s.close()
    assert off <= n // 8, "%d of %d envs left the fp64 reference" % (off, n)


def test_launch_paths_agree_bit_for_bit_with_forces(bundled_only):
    n = 512
    envs = [_make("UnitreeA1.simple", p, num_envs=n, seed=3) for p in PATHS]
    obs = [e.reset() for e in envs]
    assert all(torch.equal(obs[0], o) for o in obs[1:])
    gen = torch.Generator().manual_seed(2)
    for _ in range(6):
        x, q = _random_forces(envs[0], gen)
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        outs = []
        for e in envs:
            e.xfrc_applied.copy_(x)
            e.qfrc_applied.copy_(q)
            outs.append(e.step(act))
        for o in outs[1:]:
            for a, b in zip(outs[0][:3], o[:3]):
                assert torch.equal(a, b)
        for e in envs[1:]:
            assert torch.equal(e.xfrc_applied, envs[0].xfrc_applied)     # (the same rows zeroed by the same resets)


def test_a_push_adds_its_impulse_to_the_momentum(ref, bundled_only):
    """UnitreeA1 1 m above the floor (no contact), zero action: a horizontal force F on the trunk for one control step
    (h = n_substeps * timestep) raises the trunk_tx row of M qvel (M from the fp64 reference at each end state) by F h.
    Gravity is vertical and the motors are off, but semi-implicit Euler with implicit joint damping conserves this row only
    to first order in the step: the bound is 1 % of F h, and the fp64 reference meets it as well."""
    n, F = 8, 200.0
    env = make_env("UnitreeA1.simple", num_envs=n, seed=1)
    eng = env._get_engine()
    m, spec = env._model, env.task_spec()
    h = spec.n_substeps * m.opt_timestep
    ix, iz = m.jnt_names.index("trunk_tx"), m.jnt_names.index("trunk_tz")
    mb, tb = blobs(env)
    sim = applied_forces_ref.AppliedSim(ref, mb, tb)
    sim.reset_to(0, 10)
    q0, _ = sim.get_state()
    q0[iz] += 1.0
    v0 = np.zeros(m.nv)
    zero = np.zeros(m.nu)

    def px(q, v):
        return float((sim.forward(q, v, zero)["M"] @ v)[ix])

    eng.set_state(torch.tensor(np.tile(q0, (n, 1)), dtype=torch.float32, device="cuda"),
                  torch.zeros((n, m.nv), dtype=torch.float32, device="cuda"))
    trunk = env.body_index("trunk")
    env.xfrc_applied.zero_()
    env.xfrc_applied[:, trunk, 0] = F
    eng.step(torch.zeros((n, m.nu), device="cuda"), auto_reset=False)
    qg, vg, _ = (t.cpu().numpy().astype(np.float64) for t in eng.get_state())
    x = np.zeros((m.nbody, 6))
    x[trunk, 0] = F
    sim.set_state(q0, v0)
    qo, vo = sim.env_step(zero, xfrc=x)
    p0 = px(q0, v0)
    for q, v in ((qo, vo), (qg[0], vg[0])):
        assert abs(px(q, v) - p0 - F * h) <= 0.01 * F * h, (px(q, v) - p0, F * h)
    assert sim.lib.ref_ncon(sim.sim) == 0


def test_resets_zero_exactly_the_reset_rows(bundled_only):
    n = 128
    env = make_env("UnitreeA1.simple", num_envs=n, seed=4)
    env.reset()
    eng = env._get_engine()
    x, q = env.xfrc_applied, env.qfrc_applied
    # masked reset
    x.fill_(1.0)
    q.fill_(1.0)
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mask[::3] = 1
    eng.reset(mask=mask)
    m = mask.bool()
    assert float(x[m].abs().max()) == 0 and float(q[m].abs().max()) == 0
    assert bool((x[~m] == 1).all()) and bool((q[~m] == 1).all())
    # auto-reset: world-body rows (ignored by the physics) as markers
    gen = torch.Generator().manual_seed(6)
    seen = 0
    q.zero_()
    for _ in range(40):
        x.fill_(0.0)
        x[:, 0, :] = 1.0
        _, _, done, _ = env.step((torch.rand((n, 12), generator=gen) * 2 - 1).cuda())
        d = done.bool()
        if bool(d.any()):
            assert float(x[d].abs().max()) == 0.0
        assert bool((x[~d][:, 0] == 1).all())
        seen += int(d.sum())
    assert seen > 0, "no auto-reset happened"


def test_set_state_keeps_the_forces(bundled_only):
    env = make_env("UnitreeA1.simple", num_envs=16, seed=4)
    env.reset()
    eng = env._get_engine()
    env.qfrc_applied.fill_(0.5)
    q, v, _ = eng.get_state()
    eng.set_state(q, v)
    torch.cuda.synchronize()
    assert bool((env.qfrc_applied == 0.5).all())


def test_captured_step_reads_rewritten_forces(bundled_only):
    n, steps = 256, 8
    eager = make_env("UnitreeA1.simple", num_envs=n, seed=21)
    graphed = make_env("UnitreeA1.simple", num_envs=n, seed=21)
    assert torch.equal(eager.reset(), graphed.reset())
    eng = graphed._get_engine()
    xg, qg = graphed.xfrc_applied, graphed.qfrc_applied          # registered before the capture
    xe, qe = eager.xfrc_applied, eager.qfrc_applied
    static_act = torch.zeros((n, 12), device="cuda")
    warm = make_env("UnitreeA1.simple", num_envs=n, seed=99)
    warm.reset()
    warm._get_engine().step(static_act)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        eng.step(static_act)
    eager._get_engine().step(torch.zeros((n, 12), device="cuda"))
    graph.replay()
    gen = torch.Generator().manual_seed(5)
    pushed = 0.0
    for _ in range(steps):
        x, q = _random_forces(graphed, gen)
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        xe.copy_(x); qe.copy_(q); xg.copy_(x); qg.copy_(q)
        obs, rew, done, info = eager.step(act)
        static_act.copy_(act)
        graph.replay()
        assert torch.equal(obs, eng.obs) and torch.equal(rew, eng.reward) and torch.equal(done.view(torch.uint8), eng.done)
        pushed += float(x.abs().sum())
    assert pushed > 0


def test_two_shards_with_forces_equal_one_batch(bundled_only):
    n, steps = 64, 12
    full = make_env("UnitreeA1.simple", num_envs=n, seed=11)
    a = make_env("UnitreeA1.simple", num_envs=n // 2, seed=11, env_id_offset=0)
    b = make_env("UnitreeA1.simple", num_envs=n // 2, seed=11, env_id_offset=n // 2)
    assert torch.equal(full.reset(), torch.cat([a.reset(), b.reset()]))
    gen = torch.Generator().manual_seed(1)
    for _ in range(steps):
        x, q = _random_forces(full, gen)
        full.xfrc_applied.copy_(x); full.qfrc_applied.copy_(q)
        a.xfrc_applied.copy_(x[:n // 2]); a.qfrc_applied.copy_(q[:n // 2])
        b.xfrc_applied.copy_(x[n // 2:]); b.qfrc_applied.copy_(q[n // 2:])
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        of, rf, df, _ = full.step(act)
        oa, ra, da, _ = a.step(act[:n // 2].contiguous())
        ob, rb, db, _ = b.step(act[n // 2:].contiguous())
        assert torch.equal(of, torch.cat([oa, ob])) and torch.equal(df, torch.cat([da, db])) and torch.equal(rf, torch.cat([ra, rb]))
        assert torch.equal(full.xfrc_applied, torch.cat([a.xfrc_applied, b.xfrc_applied]))
