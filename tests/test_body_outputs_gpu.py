"""Body outputs on the GPU (include/locosim.h locosim_set_body_outputs; LocoEnv.body_state / next_body_state): registering
them changes no other bit, parity with the fp64 reference (tests/body_outputs_ref.py) at the engine's own states for every
kernel family, after steps, resets and set_state, non-finite envs, the three launch paths bit for bit, CUDA graphs,
sharding, MixedBatch members, and a push seen in the trunk's velocity."""
import os

import numpy as np
import pytest
import torch

import applied_forces_ref
from body_outputs_ref import BodyRef, compare
from full_body import make_variant
from helpers import blobs, make_env

pytestmark = pytest.mark.gpu

# launch paths of UnitreeA1 (environment variables read when an engine is created, locosim.cu setup_cfg)
PATHS = {"fused": {"LOCOSIM_RESORT": "10"}, "substeps": {"LOCOSIM_RESORT": "2"},
         "persistent": {"LOCOSIM_RESORT": "2", "LOCOSIM_PERSIST": "1"}}
# one task per kernel family: CfgEllEuler (three launch paths), CfgPyrEuler, CfgPyrRK4, CfgPyrEuler29, CfgPyrRK4_31,
# CfgPyrEuler31
FAMILIES = [("UnitreeA1.simple", "fused"), ("UnitreeA1.simple", "substeps"), ("UnitreeA1.simple", "persistent"),
            ("Talos.walk", None), ("HumanoidTorque.run", None), ("UnitreeG1.walk", None), ("Atlas.walk+arms", None),
            ("Talos.walk+arms", None)]
TOL = 2e-5          # as tests/test_body_outputs.py (the serial build of the same core)


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


def _check_rows(ref, rows, q, v, envs):
    """rows [N, nb, 13] (device) against the fp64 reference at states (q, v) [N, nv] (device), for the listed envs"""
    rows, q, v = (t.cpu().numpy() for t in (rows, q, v))
    worst = np.zeros(4)
    for i in envs:
        want = ref(q[i].astype(np.float64), v[i].astype(np.float64))
        assert np.array_equal(rows[i, 0], want[0])
        worst = np.maximum(worst, compare(rows[i], want))
    assert worst.max() < TOL, worst


@pytest.mark.parametrize("task,path", FAMILIES)
def test_registered_outputs_change_no_other_bit(oracle, bundled_only, task, path):
    """512 envs: an engine with body outputs registered steps bit for bit like one without (auto-resets included); rows of
    envs that did not reset are equal in both buffers, and next_body_state describes get_state() (the reset state where an
    env ended)."""
    n = 512
    a, b = _make(task, path, num_envs=n, seed=7), _make(task, path, num_envs=n, seed=7)
    body, nxt = b.body_state, b.next_body_state
    assert torch.equal(a.reset(), b.reset())
    ref = BodyRef(oracle, b._model)
    gen = torch.Generator().manual_seed(0)
    nu = a.info.action_space.shape[0]
    ended = 0
    for k in range(6):
        act = (torch.rand((n, nu), generator=gen) * 2 - 1).cuda()
        ra, rb = a.step(act), b.step(act)
        for x, y in zip(ra[:3], rb[:3]):
            assert torch.equal(x, y)
        assert torch.equal(ra[3]["next_obs"], rb[3]["next_obs"])
        done = rb[2].bool().cpu()
        ended += int(done.sum())
        assert torch.equal(body[~done.cuda()], nxt[~done.cuda()])
        q, v, _ = b._get_engine().get_state()
        sample = list(range(0, n, 37)) + [int(i) for i in torch.nonzero(done).flatten()[:16]]
        _check_rows(ref, nxt, q, v, sample)
    for x, y in zip(a._get_engine().get_state(), b._get_engine().get_state()):
        assert torch.equal(x, y)
    ref.close()


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "Talos.walk", "HumanoidTorque.run", "UnitreeG1.walk", "Atlas.walk+arms",
                                  "Talos.walk+arms"])
def test_body_state_matches_the_reference_at_the_returned_state(oracle, bundled_only, task):
    """auto_reset=False: the state get_state() returns is the one the step's observation describes; body_state there
    against the fp64 reference, for every family, over four steps under random actions."""
    n = 512
    env = make_variant(task, num_envs=n, seed=5)
    eng = env._get_engine()
    body = env.body_state
    eng.reset()
    ref = BodyRef(oracle, env._model)
    gen = torch.Generator().manual_seed(3)
    for k in range(4):
        act = (torch.rand((n, eng.action_dim), generator=gen) * 2 - 1).cuda()
        eng.step(act, auto_reset=False)
        q, v, _ = eng.get_state()
        # (a non-finite env is reset even without auto_reset; its body row is zeros)
        live = (body.abs().amax((1, 2)) > 0).cpu()
        _check_rows(ref, body, q, v, [i for i in range(0, n, 11) if bool(live[i])])
        assert torch.equal(body[live.cuda()], env.next_body_state[live.cuda()])
    ref.close()


def test_next_body_state_after_reset_mask_reset_obs_and_set_state(oracle, bundled_only):
    n = 128
    env = make_env("UnitreeA1.simple", num_envs=n, seed=4)
    eng = env._get_engine()
    nxt = env.next_body_state
    ref = BodyRef(oracle, env._model)
    env.reset()
    q, v, _ = eng.get_state()
    _check_rows(ref, nxt, q, v, range(0, n, 5))
    for _ in range(3):
        env.step((torch.rand((n, 12)) * 2 - 1).cuda())
    # masked reset: the masked rows are rewritten, the others keep their bits
    before = nxt.clone()
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mask[::3] = 1
    eng.reset(mask=mask)
    m = mask.bool()
    assert torch.equal(nxt[~m], before[~m]) and not torch.equal(nxt[m], before[m])
    q, v, _ = eng.get_state()
    _check_rows(ref, nxt, q, v, [int(i) for i in torch.nonzero(m).flatten()])
    # reset(obs=...): set_state underneath rewrites every row
    obs = env.step((torch.rand((n, 12)) * 2 - 1).cuda())[0].clone()
    nxt.zero_()
    env.reset(obs=obs)
    q, v, _ = eng.get_state()
    _check_rows(ref, nxt, q, v, range(n))
    # set_state
    q2, v2 = q.flip(0).contiguous(), (v * 0.5).contiguous()
    eng.set_state(q2, v2)
    _check_rows(ref, nxt, q2, v2, range(0, n, 3))
    ref.close()


def test_a_non_finite_env_gets_a_zero_body_row(oracle, bundled_only):
    """a NaN in one env's qpos (set_state: a value, not a fault): the step reports it done with all-zero obs and body rows;
    its next_body_state row describes the reset state it was given"""
    n = 64
    env = make_env("UnitreeA1.simple", num_envs=n, seed=9)
    eng = env._get_engine()
    env.reset()
    body, nxt = env.body_state, env.next_body_state
    q, v, _ = eng.get_state()
    q[5, 3] = float("nan")
    eng.set_state(q.contiguous(), v.contiguous())
    obs, _, done, _ = env.step(torch.zeros((n, 12), device="cuda"))
    assert bool(done[5]) and float(obs[5].abs().max()) == 0.0
    assert float(body[5].abs().max()) == 0.0 and bool(torch.isfinite(body).all())
    ref = BodyRef(oracle, env._model)
    q, v, _ = eng.get_state()
    _check_rows(ref, nxt, q, v, [5, 6])
    ref.close()


def test_launch_paths_agree_bit_for_bit(bundled_only):
    n = 512
    envs = [_make("UnitreeA1.simple", p, num_envs=n, seed=3) for p in PATHS]
    for e in envs:
        e.body_state
    obs = [e.reset() for e in envs]
    assert all(torch.equal(obs[0], o) for o in obs[1:])
    gen = torch.Generator().manual_seed(2)
    resets = 0
    for _ in range(8):
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        outs = [e.step(act) for e in envs]
        resets += int(outs[0][2].bool().sum())
        for e, o in zip(envs[1:], outs[1:]):
            assert torch.equal(outs[0][2], o[2])
            assert torch.equal(envs[0].body_state, e.body_state) and torch.equal(envs[0].next_body_state, e.next_body_state)
    assert resets > 0


def test_captured_step_writes_the_registered_buffers(bundled_only):
    n, steps = 256, 8
    eager = make_env("UnitreeA1.simple", num_envs=n, seed=21)
    graphed = make_env("UnitreeA1.simple", num_envs=n, seed=21)
    be, ne = eager.body_state, eager.next_body_state
    bg, ng = graphed.body_state, graphed.next_body_state          # registered before the capture
    assert torch.equal(eager.reset(), graphed.reset())
    eng = graphed._get_engine()
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
    for _ in range(steps):
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        eager.step(act)
        static_act.copy_(act)
        bg.zero_()
        ng.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(be, bg) and torch.equal(ne, ng) and float(bg.abs().max()) > 0


def test_two_shards_equal_one_batch(bundled_only):
    n, steps = 64, 10
    full = make_env("UnitreeA1.simple", num_envs=n, seed=11)
    a = make_env("UnitreeA1.simple", num_envs=n // 2, seed=11, env_id_offset=0)
    b = make_env("UnitreeA1.simple", num_envs=n // 2, seed=11, env_id_offset=n // 2)
    for e in (full, a, b):
        e.next_body_state
    assert torch.equal(full.reset(), torch.cat([a.reset(), b.reset()]))
    assert torch.equal(full.next_body_state, torch.cat([a.next_body_state, b.next_body_state]))
    gen = torch.Generator().manual_seed(1)
    for _ in range(steps):
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        full.step(act)
        a.step(act[:n // 2].contiguous())
        b.step(act[n // 2:].contiguous())
        assert torch.equal(full.body_state, torch.cat([a.body_state, b.body_state]))
        assert torch.equal(full.next_body_state, torch.cat([a.next_body_state, b.next_body_state]))


def test_mixed_batch_members_expose_their_own_rows(bundled_only):
    from loco_mujoco_b200.parallel import MixedBatch
    n = 48
    mb = MixedBatch([("Atlas.walk.real", n, {}), ("Talos.walk.real", n, {})], device="cuda:0", seed=3, debug=True)
    solo = [make_env("Atlas.walk", num_envs=n, seed=3, env_id_offset=0), make_env("Talos.walk", num_envs=n, seed=3, env_id_offset=n)]
    for e in mb.envs + solo:
        e.body_state
    mb.reset()
    for e in solo:
        e.reset()
    gen = torch.Generator().manual_seed(4)
    for _ in range(4):
        acts = [(torch.rand((n, e.action_dim), generator=gen) * 2 - 1).cuda() for e in mb.engines]
        mb.step(acts)
        for e, a in zip(solo, acts):
            e.step(a)
        torch.cuda.synchronize()
        for m, s in zip(mb.envs, solo):
            assert m.body_state.shape[1] == s._model.nbody
            assert torch.equal(m.body_state, s.body_state) and torch.equal(m.next_body_state, s.next_body_state)


def test_a_push_shows_in_the_trunk_velocity(oracle, bundled_only):
    """UnitreeA1 1 m above the floor at rest, zero action, a horizontal force F on the trunk's CoM for one control step
    (h = n_substeps * timestep): the trunk's linear x velocity in body_state is positive and close to F h / M (M the
    robot's mass: the momentum F h spreads over the whole robot; within 15 %, as the legs swing back against their joint
    damping), and it matches the fp64 reference at the state the fp64 applied-force reference reaches (2e-3, the state
    tolerance of test_gpu_parity)."""
    n, F = 8, 200.0
    env = make_env("UnitreeA1.simple", num_envs=n, seed=1)
    eng = env._get_engine()
    m, spec = env._model, env.task_spec()
    h = spec.n_substeps * m.opt_timestep
    iz = m.jnt_names.index("trunk_tz")
    trunk = env.body_index("trunk")
    sim = applied_forces_ref.AppliedSim(applied_forces_ref.load(), *blobs(env))
    sim.reset_to(0, 10)
    q0, _ = sim.get_state()
    q0[iz] += 1.0
    eng.set_state(torch.tensor(np.tile(q0, (n, 1)), dtype=torch.float32, device="cuda"),
                  torch.zeros((n, m.nv), dtype=torch.float32, device="cuda"))
    body = env.body_state
    env.xfrc_applied.zero_()
    env.xfrc_applied[:, trunk, 0] = F
    eng.step(torch.zeros((n, m.nu), device="cuda"), auto_reset=False)
    vx = body[:, trunk, 10].cpu().numpy()
    mass = float(np.sum(m.body_mass))
    assert np.all(vx > 0) and np.all(np.abs(vx - F * h / mass) <= 0.15 * F * h / mass), (vx, F * h / mass)
    x = np.zeros((m.nbody, 6))
    x[trunk, 0] = F
    sim.set_state(q0, np.zeros(m.nv))
    qo, vo = sim.env_step(np.zeros(m.nu), xfrc=x)
    want = BodyRef(oracle, m)(qo, vo)
    assert abs(vx[0] - want[trunk, 10]) <= 2e-3 * (1 + abs(want[trunk, 10])), (vx[0], want[trunk, 10])
    sim.close()


@pytest.mark.parametrize("task,path", FAMILIES + [("Atlas.carry", None), ("Talos.carry", None)])
def test_terminal_rows_of_auto_reset_envs(oracle, bundled_only, task, path):
    """The d_body rows of envs a step ends and auto-resets describe their terminal state. In lock-step from the same state,
    a twin engine steps with auto_reset=False and keeps that state: body_state of the two is equal bit for bit, and for the
    ended, finite envs it matches the fp64 reference at the twin's get_state(). The twin then resets exactly those envs
    (the same counter-based draws as the auto-reset) and the two engines agree again bit for bit, state and next_body_state
    included. The carry tasks give every env its own parameter-pool row (the carried weight), which a reset redraws."""
    n = 512
    a, b = _make(task, path, num_envs=n, seed=13), _make(task, path, num_envs=n, seed=13)
    ea, eb = a._get_engine(), b._get_engine()
    ba, bb, na, nb = a.body_state, b.body_state, a.next_body_state, b.next_body_state
    assert torch.equal(ea.reset(), eb.reset())
    ref = BodyRef(oracle, b._model)
    gen = torch.Generator().manual_seed(8)
    ended = 0
    for k in range(8):
        act = (torch.rand((n, ea.action_dim), generator=gen) * 2 - 1).cuda()
        _, _, da, _ = ea.step(act, auto_reset=True)
        _, _, db, _ = eb.step(act, auto_reset=False)
        assert torch.equal(da, db)
        assert torch.equal(ba, bb)
        done = da.bool()
        bad = bb.abs().amax((1, 2)) == 0                      # non-finite: zero rows, reset by both engines
        finite_done = torch.nonzero(done & ~bad).flatten().cpu()
        ended += len(finite_done)
        if len(finite_done):
            q, v, _ = eb.get_state()
            _check_rows(ref, bb, q, v, [int(i) for i in finite_done[:24]])
            eb.reset(mask=(done & ~bad).to(torch.uint8))
        for x, y in zip(ea.get_state(), eb.get_state()):
            assert torch.equal(x, y)
        assert torch.equal(na, nb)
    ref.close()
    assert ended > 0, "no env ended: the terminal rows were not exercised"


def test_a_graph_captured_before_registering_is_captured_again(bundled_only):
    """A step captured while nothing is registered does not write the rows (include/locosim.h). Registering, replaying that
    old graph anyway, then capturing again: from the first replay of the new graph on, every row equals an eager twin's,
    so nothing the old graph left behind (its reset marks) hides a row."""
    n, steps = 256, 8
    eager = make_env("UnitreeA1.simple", num_envs=n, seed=31)
    graphed = make_env("UnitreeA1.simple", num_envs=n, seed=31)
    be, ne = eager.body_state, eager.next_body_state
    assert torch.equal(eager.reset(), graphed.reset())
    eng, eeng = graphed._get_engine(), eager._get_engine()
    static_act = torch.zeros((n, 12), device="cuda")
    warm = make_env("UnitreeA1.simple", num_envs=n, seed=99)
    warm.reset()
    warm._get_engine().step(static_act)
    torch.cuda.synchronize()
    old = torch.cuda.CUDAGraph()
    with torch.cuda.graph(old):                               # nothing registered
        eng.step(static_act)
    gen = torch.Generator().manual_seed(6)

    def both(graph):
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        eeng.step(act)
        static_act.copy_(act)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(eeng.done, eng.done)

    for _ in range(3):
        both(old)
    bg, ng = graphed.body_state, graphed.next_body_state      # first access: registered now
    resets = 0
    for _ in range(4):                                        # the old graph after registering: marks, few rows
        both(old)
        resets += int(eng.done.bool().sum())
    assert resets > 0
    new = torch.cuda.CUDAGraph()
    with torch.cuda.graph(new):
        eng.step(static_act)
    for _ in range(steps):
        bg.fill_(-1.0)
        ng.fill_(-1.0)
        both(new)
        assert torch.equal(be, bg) and torch.equal(ne, ng)
