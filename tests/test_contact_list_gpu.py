"""Contact list on the GPU (include/locosim.h locosim_set_contact_list_outputs; LocoEnv.contacts): parity with the fp64
reference's last sub-step (tests/contact_list_ref.py) from the engine's own pre-step states on every kernel family and launch
path, registering changes no other bit, the launch paths bit for bit, identities with the contact outputs and the foot-force
observation, self contacts, terminal rows of auto-reset envs, non-finite envs, the calls that must not write, CUDA graphs,
sharding, MixedBatch members and saved-state replay."""
import os

import numpy as np
import pytest
import torch

import contact_list_ref as clr
import contact_wrench_ref as cwr
from full_body import make_variant
from helpers import blobs, make_env

pytestmark = pytest.mark.gpu

# launch paths (environment variables read when an engine is created, locosim.cu setup_cfg)
PATHS = {"fused": {"LOCOSIM_RESORT": "10"}, "substeps": {"LOCOSIM_RESORT": "2"},
         "persistent": {"LOCOSIM_RESORT": "2", "LOCOSIM_PERSIST": "1"}}
# one task per kernel family on each launch path: CfgEllEuler (UnitreeA1, elliptic cones), CfgPyrEuler (Talos), CfgPyrRK4
# (HumanoidTorque), CfgPyrEuler29 (UnitreeG1), CfgPyrRK4_31 (Atlas with arms), CfgPyrEuler31 (Talos with arms), all pyramidal
FAMILIES = [(t, p) for t in ("UnitreeA1.simple", "Talos.walk", "HumanoidTorque.run", "UnitreeG1.walk", "Atlas.walk+arms",
                             "Talos.walk+arms") for p in PATHS]


@pytest.fixture(scope="module")
def ref():
    return cwr.load()


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


def _bufs(env):
    """the registered (ncon, con, con_id) tensors of env.contacts"""
    env.contacts
    return env._contact_list[:3]


def _snap(env):
    return tuple(x.clone() for x in _bufs(env))


def _equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def _rows_ok(bufs):
    ncon, con, con_id = bufs
    C = con.shape[1]
    past = torch.arange(C, device=con.device)[None, :] >= ncon[:, None].long()
    return bool((ncon >= 0).all() and (ncon <= C).all() and (con[past] == 0).all() and (con_id[past] == -1).all()
                and (con_id[~past] >= 0).all())


def _act(gen, n, nu):
    return (torch.rand((n, nu), generator=gen) * 2 - 1).cuda()


@pytest.mark.parametrize("task,path", FAMILIES)
def test_matches_the_reference_and_changes_no_other_bit(ref, bundled_only, task, path):
    """512 envs, three engines from one seed: (a) body, contact, dof and reference outputs registered, (b) the same plus the
    contact list, (c) the contact list alone. a and b step bit for bit alike in every output, b's and c's lists are equal
    bit for bit, and sampled rows match the fp64 reference's last sub-step from the engine's own pre-step state and warm
    start within clr.TOL (or within 10x the oracle's own change under an fp32-sized perturbation, where a contact switches
    within the step)."""
    n = 512
    a, b, c = (_make(task, path, num_envs=n, seed=7, truncate_at_trajectory_end=True) for _ in range(3))
    for e in (a, b):
        e.body_state, e.contact_wrench, e.dof_outputs, e.reference_body_state
    lb, lc = _bufs(b), _bufs(c)
    oa = a.reset()
    assert torch.equal(oa, b.reset()) and torch.equal(oa, c.reset())
    others = lambda e: (e.body_state, e.next_body_state, e.contact_wrench, e.dof_outputs, e.reference_body_state,  # noqa
                        e.next_reference_body_state)
    eng = b._get_engine()
    mb, tb = blobs(b)
    m = b._model
    user = b._model_user_features[0]
    gen = torch.Generator().manual_seed(0)
    nu = a.info.action_space.shape[0]
    checked, allowed, touched = 0, 0, 0
    for k in range(4):
        act = _act(gen, n, nu)
        q0, v0, w0 = (x.cpu().numpy().astype(np.float64) for x in eng.get_state())
        ra, rb, rc = a.step(act), b.step(act), c.step(act)
        for x, y, z in zip(ra[:3], rb[:3], rc[:3]):
            assert torch.equal(x, y) and torch.equal(x, z)
        assert torch.equal(ra[3]["next_obs"], rb[3]["next_obs"]) and torch.equal(ra[3]["next_obs"], rc[3]["next_obs"])
        assert all(torch.equal(x, y) for x, y in zip(others(a), others(b)))
        assert _equal(lb, lc) and _rows_ok(lb)
        ncon, con, con_id = (x.cpu().numpy() for x in lb)
        an = act.cpu().numpy().astype(np.float64)
        for i in range(k, n, 43):
            oe = ref.env(mb, tb)
            oe.set_user(user)
            oe.set_state(q0[i], v0[i], w0[i])
            cwr.env_step(ref, oe, an[i])
            want = clr.reference(ref, oe.sim, m)
            oe.close()
            got = clr.unpack(ncon[i], con[i], con_id[i])
            touched += int(len(want["dist"]) > 0 and np.abs(want["force"]).max() > 1.0)
            err = clr.mismatch(got, want)
            if err > 1.0:
                gap = clr.sensitivity(ref, mb, tb, m, q0[i], v0[i], an[i], want, warmstart=w0[i], user=user)
                assert err < 10 * gap, (task, path, k, i, err, gap)
                allowed += 1
            checked += 1
    for x, y in zip(a._get_engine().get_state(), eng.get_state()):
        assert torch.equal(x, y)
    assert touched > checked // 4, (touched, checked)
    assert allowed <= max(2, checked // 20), (allowed, checked)


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "HumanoidTorque.run", "Atlas.walk+arms"])
def test_launch_paths_agree_bit_for_bit(bundled_only, task):
    n = 512
    envs = [_make(task, p, num_envs=n, seed=3) for p in PATHS]
    obs = [e.reset() for e in envs]
    assert all(torch.equal(obs[0], o) for o in obs[1:])
    gen = torch.Generator().manual_seed(2)
    nu = envs[0].info.action_space.shape[0]
    resets = 0
    for _ in range(8):
        act = _act(gen, n, nu)
        outs = [e.step(act) for e in envs]
        resets += int(outs[0][2].bool().sum())
        for e, o in zip(envs[1:], outs[1:]):
            assert torch.equal(outs[0][0], o[0])
            assert _equal(_bufs(envs[0]), _bufs(e))
    assert resets > 0 and int(_bufs(envs[0])[0].max()) > 0


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "Talos.walk", "HumanoidTorque.run"])
def test_one_sub_step_sums_to_the_contact_outputs(bundled_only, task):
    """n_substeps = 1: the list and the contact outputs describe the same evaluation, so summing the list per body with the
    contact outputs' signs gives contact_wrench's forces (and, for Euler, whose evaluation is at the step's start state,
    the torques about the start state's xpos, next_body_state before the step) to fp32 rounding."""
    n = 256
    env = make_env(task, num_envs=n, seed=5, n_substeps=1)
    nb, rk4 = env._model.nbody, env._model.opt_integrator == 1
    cw, nxt, c = env.contact_wrench, env.next_body_state, env.contacts
    env.reset()
    gen = torch.Generator().manual_seed(6)
    nu = env.info.action_space.shape[0]
    seen = 0
    for _ in range(6):
        xpos = nxt[:, :, 0:3].double().clone()
        env._get_engine().step(_act(gen, n, nu), auto_reset=False)
        assert _rows_ok(_bufs(env))
        valid = torch.arange(c.dist.shape[1], device="cuda")[None, :] < c.ncon[:, None].long()
        fr, f = c.frame.double(), c.force.double()
        F = (f[..., 0:3, None] * fr).sum(-2)                                  # f0 n + f1 t1 + f2 t2
        T = (f[..., 3:6, None] * fr).sum(-2)
        w = torch.zeros((n, nb, 6), dtype=torch.float64, device="cuda")
        for side, s in ((0, -1.0), (1, 1.0)):
            b = c.body[..., side].long().clamp(min=0)
            r = c.pos.double() - torch.gather(xpos, 1, b[..., None].expand(-1, -1, 3))
            wr = torch.cat([F, torch.cross(r, F, dim=-1) + T], -1) * (s * valid * (b > 0))[..., None]
            w.scatter_add_(1, b[..., None].expand(-1, -1, 6), wr)
        scale = 1e-5 * max(1.0, float(cw.abs().max()))
        assert float((w[..., :3] - cw[..., :3].double()).abs().max()) < scale
        if not rk4:
            assert float((w[..., 3:] - cw[..., 3:].double()).abs().max()) < 10 * scale
        seen += int(valid.sum())
    assert seen > n


def test_foot_forces_are_the_first_floor_contacts(bundled_only):
    """use_foot_forces with n_substeps = 1: each foot group's observation is the force of its first floor contact in the list
    (the engine's "first contact") times float32(1 / 1000), bit for bit; zero where the group has none"""
    from loco_mujoco_b200.task import GRF_FLOOR
    n = 256
    env = make_env("UnitreeA1.simple", num_envs=n, seed=8, n_substeps=1, use_foot_forces=True,
                   use_absorbing_states=False)
    spec = env.task_spec()
    grp = torch.tensor(np.asarray(spec.grf_group), dtype=torch.long, device="cuda")
    n_grf = spec.n_grf
    c = env.contacts
    env.reset()
    gen = torch.Generator().manual_seed(9)
    hits = 0
    for _ in range(6):
        obs, _, _, _ = env._get_engine().step(_act(gen, n, 12), auto_reset=False)
        g = c.geom.long().clamp(min=0)
        g1, g2 = grp[g[..., 0]], grp[g[..., 1]]
        valid = torch.arange(c.dist.shape[1], device="cuda")[None, :] < c.ncon[:, None].long()
        grf = obs[:, -3 * n_grf:].view(n, n_grf, 3)
        for k in range(n_grf):
            hit = valid & (((g1 == GRF_FLOOR) & (g2 == k)) | ((g2 == GRF_FLOOR) & (g1 == k)))
            first = torch.where(hit, torch.arange(hit.shape[1], device="cuda")[None, :], hit.shape[1]).min(dim=1).values
            has = first < hit.shape[1]
            f = c.force[torch.arange(n, device="cuda"), first.clamp(max=hit.shape[1] - 1), 0:3]
            want = torch.where(has[:, None], f * torch.tensor(1.0 / 1000.0, dtype=torch.float32, device="cuda"),
                               torch.zeros_like(f))
            assert torch.equal(grf[:, k], want), k
            hits += int(has.sum())
    assert hits > n


def test_self_contacts_name_two_bodies(ref, bundled_only):
    """HumanoidTorque at reset-table poses with the joints bent at random until bones interpenetrate (as the contact-wrench
    tests find self contacts): contacts between two non-world geoms carry two non-zero bodies, floor contacts the world
    as body1, and the bodies are geom_bodyid of the geoms"""
    n = 512
    env = make_env("HumanoidTorque.run", num_envs=n, seed=2)
    m, spec = env._model, env.task_spec()
    eng = env._get_engine()
    c = env.contacts
    env.reset()
    table = spec.table.reshape(-1, spec.table.shape[-1])
    rng = np.random.RandomState(3)
    rows = table[rng.randint(len(table), size=n)]
    q, v = rows[:, :m.nv].copy(), rows[:, m.nv:2 * m.nv].copy()
    q[:, 6:] += rng.uniform(-1.2, 1.2, (n, m.nv - 6))
    eng.set_state(torch.tensor(q, dtype=torch.float32, device="cuda"), torch.tensor(v, dtype=torch.float32, device="cuda"))
    eng.step(torch.zeros((n, m.nu), device="cuda"), auto_reset=False)
    valid = (torch.arange(c.dist.shape[1], device="cuda")[None, :] < c.ncon[:, None].long()).cpu().numpy()
    geom, body = c.geom.cpu().numpy()[valid], c.body.cpu().numpy()[valid]
    assert np.array_equal(body, np.asarray(m.geom_bodyid)[geom])
    world = np.asarray(m.geom_bodyid)[geom[:, 0]] == 0
    assert np.all(body[~world] > 0) and np.all(body[world][:, 1] > 0)
    assert int((~world).sum()) > 0, "no self contacts"


@pytest.mark.parametrize("task,path", [("UnitreeA1.simple", p) for p in PATHS] + [("Atlas.walk+arms", None)])
def test_terminal_rows_of_auto_reset_envs(bundled_only, task, path):
    """In lock-step from the same state, a twin engine steps with auto_reset=False: the lists are equal bit for bit, those of
    the envs the first one ended and reset included."""
    n = 512
    a, b = _make(task, path, num_envs=n, seed=13), _make(task, path, num_envs=n, seed=13)
    ea, eb = a._get_engine(), b._get_engine()
    la, lb = _bufs(a), _bufs(b)
    assert torch.equal(ea.reset(), eb.reset())
    gen = torch.Generator().manual_seed(8)
    ended = 0
    for _ in range(8):
        act = _act(gen, n, ea.action_dim)
        _, _, da, _ = ea.step(act, auto_reset=True)
        _, _, db, _ = eb.step(act, auto_reset=False)
        assert torch.equal(da, db) and _equal(la, lb)
        done = da.bool()
        ended += int(done.sum())
        if bool(done.any()):
            q, _, _ = eb.get_state()
            fin = torch.isfinite(q).all(dim=1)
            eb.reset(mask=(done & fin).to(torch.uint8))
        for x, y in zip(ea.get_state(), eb.get_state()):
            assert torch.equal(x, y)
    assert ended > 0, "no env ended: the terminal rows were not exercised"


def test_non_finite_env_and_the_calls_that_do_not_write(bundled_only):
    """a NaN in one env's qpos (set_state: a value, not a fault) gives ncon = 0 and empty rows on every launch path; reset(),
    set_state() and load_state() leave the rows alone"""
    for path in PATHS:
        n = 64
        env = _make("UnitreeA1.simple", path, num_envs=n, seed=9)
        eng = env._get_engine()
        env.reset()
        bufs = _bufs(env)
        for x in bufs:
            x.fill_(7)
        q, v, _ = eng.get_state()
        q[5, 3] = float("nan")
        eng.set_state(q.contiguous(), v.contiguous())
        obs, _, done, _ = env.step(torch.zeros((n, 12), device="cuda"))
        assert bool(done[5]) and float(obs[5].abs().max()) == 0.0
        assert int(bufs[0][5]) == 0 and _rows_ok(bufs)
        assert int(bufs[0].max()) > 0
        rows = env.save_state()
        env.step(torch.zeros((n, 12), device="cuda"))
        keep = _snap(env)
        env.reset()
        q, v, _ = eng.get_state()
        eng.set_state(q, v)
        env.load_state(rows)
        torch.cuda.synchronize()
        assert _equal(keep, bufs)


def test_graphs_captured_before_and_after_registering(bundled_only):
    """the step kernels read the registration when they run: a graph captured while nothing was registered writes the
    list at replays after the registration, as eager steps do; registering None stops it"""
    n, steps = 256, 6
    eager = make_env("UnitreeA1.simple", num_envs=n, seed=21)
    early = make_env("UnitreeA1.simple", num_envs=n, seed=21)
    le = _bufs(eager)
    assert torch.equal(eager.reset(), early.reset())
    warm = make_env("UnitreeA1.simple", num_envs=n, seed=99)
    warm.reset()
    static_act = torch.zeros((n, 12), device="cuda")
    warm._get_engine().step(static_act)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                               # nothing registered yet
        early._get_engine().step(static_act)
    lg = _bufs(early)                                           # registered after the capture
    eager._get_engine().step(torch.zeros((n, 12), device="cuda"))
    graph.replay()
    torch.cuda.synchronize()
    assert _equal(le, lg)
    after = torch.cuda.CUDAGraph()                              # and one captured with the list registered
    twin = make_env("UnitreeA1.simple", num_envs=n, seed=21)
    lt = _bufs(twin)
    twin.reset()
    twin._get_engine().step(torch.zeros((n, 12), device="cuda"))
    torch.cuda.synchronize()
    with torch.cuda.graph(after):
        twin._get_engine().step(static_act)
    gen = torch.Generator().manual_seed(5)
    for _ in range(steps):
        act = _act(gen, n, 12)
        eager.step(act)
        static_act.copy_(act)
        for x in lg + lt:
            x.zero_()
        graph.replay()
        after.replay()
        torch.cuda.synchronize()
        assert _equal(le, lg) and _equal(le, lt) and int(lg[0].max()) > 0
    early._get_engine().set_contact_list_outputs()
    for x in lg:
        x.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(float(x.abs().max()) == 0 for x in lg)


def test_two_shards_equal_one_batch(bundled_only):
    n, steps = 64, 6
    full = make_env("UnitreeA1.simple", num_envs=n, seed=11)
    a = make_env("UnitreeA1.simple", num_envs=n // 2, seed=11, env_id_offset=0)
    b = make_env("UnitreeA1.simple", num_envs=n // 2, seed=11, env_id_offset=n // 2)
    assert torch.equal(full.reset(), torch.cat([a.reset(), b.reset()]))
    gen = torch.Generator().manual_seed(1)
    for _ in range(steps):
        act = _act(gen, n, 12)
        full.step(act)
        a.step(act[:n // 2].contiguous())
        b.step(act[n // 2:].contiguous())
        assert all(torch.equal(x, torch.cat([y, z])) for x, y, z in zip(_bufs(full), _bufs(a), _bufs(b)))


def test_mixed_batch_members_expose_their_own_rows(bundled_only):
    from loco_mujoco_b200.parallel import MixedBatch
    n = 48
    mb = MixedBatch([("Atlas.walk.real", n, {}), ("Talos.walk.real", n, {})], device="cuda:0", seed=3, debug=True)
    solo = [make_env("Atlas.walk", num_envs=n, seed=3, env_id_offset=0), make_env("Talos.walk", num_envs=n, seed=3, env_id_offset=n)]
    for e in mb.envs + solo:
        e.contacts
    mb.reset()
    for e in solo:
        e.reset()
    gen = torch.Generator().manual_seed(4)
    for _ in range(4):
        acts = [_act(gen, n, e.action_dim) for e in mb.engines]
        mb.step(acts)
        for e, a in zip(solo, acts):
            e.step(a)
        torch.cuda.synchronize()
        for m, s in zip(mb.envs, solo):
            assert _equal(_bufs(m), _bufs(s))
    assert int(_bufs(mb.envs[0])[0].max()) > 0


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "HumanoidTorque.run"])
def test_saved_state_replay_reproduces_the_list(bundled_only, task):
    """save, run 6 steps recording the lists, load the rows back, run the same actions again: the same lists bit for bit,
    auto-resets included"""
    n = 256
    env = make_env(task, num_envs=n, seed=17)
    env.contacts
    env.reset()
    nu = env.info.action_space.shape[0]
    gen = torch.Generator().manual_seed(3)
    for _ in range(3):
        env.step(_act(gen, n, nu))
    rows = env.save_state()
    acts = [_act(gen, n, nu) for _ in range(6)]
    first = []
    for a in acts:
        env.step(a)
        first.append(_snap(env))
    env.load_state(rows)
    for a, want in zip(acts, first):
        env.step(a)
        assert _equal(_bufs(env), want)
    assert any(int(w[0].max()) > 0 for w in first)
