"""Reference outputs on the GPU (include/locosim.h locosim_set_reference_outputs / locosim_create_dataset_bodies;
LocoEnv.reference_body_state / next_reference_body_state / create_dataset_bodies): registering changes no other bit, the rows
equal the body outputs of a twin engine reset onto the same table row, terminal rows, non-finite envs, the three launch
paths bit for bit, CUDA graphs, sharding, MixedBatch members, the dataset, and a DeepMimic end-effector term as the usage
example."""
import os

import pytest
import torch

from full_body import make_variant
from helpers import make_env

pytestmark = pytest.mark.gpu

# launch paths of UnitreeA1 (environment variables read when an engine is created, locosim.cu setup_cfg)
PATHS = {"fused": {"LOCOSIM_RESORT": "10"}, "substeps": {"LOCOSIM_RESORT": "2"},
         "persistent": {"LOCOSIM_RESORT": "2", "LOCOSIM_PERSIST": "1"}}
# one task per kernel family: CfgEllEuler (three launch paths), CfgPyrEuler, CfgPyrRK4, CfgPyrEuler29, CfgPyrRK4_31,
# CfgPyrEuler31
FAMILIES = [("UnitreeA1.simple", "fused"), ("UnitreeA1.simple", "substeps"), ("UnitreeA1.simple", "persistent"),
            ("Talos.walk", None), ("HumanoidTorque.run", None), ("UnitreeG1.walk", None), ("Atlas.walk+arms", None),
            ("Talos.walk+arms", None)]
N = 512
# the reference follows the cursor, which moves only under the tracking reward or the end-of-trajectory limit
KW = dict(truncate_at_trajectory_end=True)


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
    kw = dict(KW, **kw)
    env = _with_env(PATHS[path] if path else {}, lambda: make_variant(task, **kw))
    _with_env(PATHS[path] if path else {}, env._get_engine)
    return env


def _act(gen, n, nu):
    return (torch.rand((n, nu), generator=gen) * 2 - 1).cuda()


def _twin_rows(task, cursor, angle=None, **kw):
    """next_body_state of a fresh engine reset onto the table rows `cursor` [n] (traj * T + sample) with pinned angles"""
    twin = make_variant(task, num_envs=len(cursor), **dict(KW, **kw))
    eng = twin._get_engine()
    nxt = twin.next_body_state
    T = twin.trajectories.trajectory_length
    c = cursor.to(torch.int32)
    eng.reset(traj_no=(c // T).contiguous(), step_no=(c % T).contiguous(), rot_angle=angle)
    torch.cuda.synchronize()
    return nxt.clone()


@pytest.mark.parametrize("task,path", FAMILIES)
def test_registering_changes_no_other_bit(bundled_only, task, path):
    """Two engines with body outputs registered, one of them with reference outputs too: every output, the body outputs
    included, and the state are equal bit for bit over steps with auto-resets. Rows of envs that did not reset are equal in
    both reference buffers, and for envs a step reset the reference of the state to act on next IS its body state."""
    a, b = _make(task, path, num_envs=N, seed=7), _make(task, path, num_envs=N, seed=7)
    for e in (a, b):
        e.body_state
    ref, nref = b.reference_body_state, b.next_reference_body_state
    assert torch.equal(a.reset(), b.reset())
    assert torch.equal(a.next_body_state, b.next_body_state)
    gen = torch.Generator().manual_seed(0)
    nu = a.info.action_space.shape[0]
    ended = 0
    for _ in range(6):
        act = _act(gen, N, nu)
        ra, rb = a.step(act), b.step(act)
        for x, y in zip(ra[:3], rb[:3]):
            assert torch.equal(x, y)
        assert torch.equal(ra[3]["next_obs"], rb[3]["next_obs"])
        assert torch.equal(a.body_state, b.body_state) and torch.equal(a.next_body_state, b.next_body_state)
        done = (rb[2] | rb[3]["truncated"]).bool()
        ended += int(done.sum())
        assert torch.equal(ref[~done], nref[~done])
        assert torch.equal(nref[done], b.next_body_state[done])
    for x, y in zip(a._get_engine().get_state(), b._get_engine().get_state()):
        assert torch.equal(x, y)
    assert ended > 0


@pytest.mark.parametrize("rot", [False, True])
def test_next_reference_equals_next_body_state_after_reset(bundled_only, rot):
    kw = dict(setup_random_rot=True) if rot else {}
    env = _make("UnitreeA1.simple", num_envs=N, seed=4, **kw)
    nxt, nref = env.next_body_state, env.next_reference_body_state
    env.reset()
    assert torch.equal(nxt, nref) and float(nref.abs().max()) > 0
    gen = torch.Generator().manual_seed(1)
    for _ in range(3):
        env.step(_act(gen, N, 12))
    mask = torch.zeros(N, dtype=torch.uint8, device="cuda")
    mask[::3] = 1
    before = nref.clone()
    env._get_engine().reset(mask=mask)
    m = mask.bool()
    assert torch.equal(nref[m], nxt[m]) and torch.equal(nref[~m], before[~m])
    # set_state moves no cursor and does not write the reference
    q, v, _ = env._get_engine().get_state()
    env._get_engine().set_state(q.flip(0).contiguous(), v.contiguous())
    assert torch.equal(nref[~m], before[~m]) and not torch.equal(nxt, nref)


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("rot", [False, True])
def test_next_reference_equals_a_twin_reset_onto_the_cursor(bundled_only, path, rot):
    """After K steps, each env's next_reference_body_state equals, bit for bit, next_body_state of a twin engine reset onto
    the same table row (cursor()) with the same angle. Under setup_random_rot the angles are pinned at the first reset, so the
    envs compared are those no step has reset since."""
    kw = dict(setup_random_rot=True) if rot else {}
    env = _make("UnitreeA1.simple", path, num_envs=N, seed=9, **kw)
    eng = env._get_engine()
    nref = env.next_reference_body_state
    angle = torch.rand(N, generator=torch.Generator().manual_seed(3)).cuda() * 6.2831853 if rot else None
    eng.reset(rot_angle=angle)
    gen = torch.Generator().manual_seed(2)
    fresh = torch.ones(N, dtype=torch.bool, device="cuda")
    for _ in range(12):
        _, _, done, info = env.step(_act(gen, N, 12))
        fresh &= ~(done | info["truncated"]).bool()
    want = _twin_rows("UnitreeA1.simple", eng.cursor(), angle, **kw)
    keep = fresh if rot else torch.ones_like(fresh)
    assert int(keep.sum()) > N // 4
    assert torch.equal(nref[keep], want[keep])
    T = env.trajectories.trajectory_length
    assert bool(((eng.cursor() % T) > 0).any())                # the cursors have moved


@pytest.mark.parametrize("task,path", [("UnitreeA1.simple", "fused"), ("UnitreeA1.simple", "persistent"),
                                       ("HumanoidTorque.run", None), ("Talos.walk+arms", None)])
def test_terminal_rows_equal_an_auto_reset_false_twin(bundled_only, task, path):
    """In lock-step from the same state, a twin steps with auto_reset=False: for every env a step ends, the reference row of
    the returned state (d_ref) is equal bit for bit in both. The twin then resets exactly those envs and the two agree
    again, next_reference_body_state included."""
    a, b = _make(task, path, num_envs=N, seed=13), _make(task, path, num_envs=N, seed=13)
    ea, eb = a._get_engine(), b._get_engine()
    ra, rb, na, nb = a.reference_body_state, b.reference_body_state, a.next_reference_body_state, b.next_reference_body_state
    assert torch.equal(ea.reset(), eb.reset())
    gen = torch.Generator().manual_seed(8)
    ended = 0
    for _ in range(10):
        act = _act(gen, N, ea.action_dim)
        _, _, da, _ = ea.step(act, auto_reset=True)
        _, _, db, _ = eb.step(act, auto_reset=False)
        assert torch.equal(da, db)
        assert torch.equal(ra, rb)
        done = da != 0
        ended += int(done.sum())
        if bool(done.any()):
            eb.reset(mask=done.to(torch.uint8))
        for x, y in zip(ea.get_state(), eb.get_state()):
            assert torch.equal(x, y)
        assert torch.equal(ea.cursor(), eb.cursor()) and torch.equal(na, nb)
    assert ended > 0


def test_non_finite_envs_give_zero_rows(bundled_only):
    for auto in (True, False):
        env = _make("UnitreeA1.simple", num_envs=64, seed=2)
        eng = env._get_engine()
        ref, nref, nxt = env.reference_body_state, env.next_reference_body_state, env.next_body_state
        env.reset()
        q, v, _ = eng.get_state()
        q[5, 3] = float("nan")
        eng.set_state(q.contiguous(), v.contiguous())
        obs, _, done, _ = eng.step(torch.zeros((64, 12), device="cuda"), auto_reset=auto)
        assert bool(done[5]) and float(obs[5].abs().max()) == 0.0
        assert float(ref[5].abs().max()) == 0.0 and bool(torch.isfinite(ref).all())
        assert float(ref[6].abs().max()) > 0
        assert torch.equal(nref[5], nxt[5]) and float(nref[5].abs().max()) > 0      # the reset's reference


def test_launch_paths_agree_bit_for_bit(bundled_only):
    envs = [_make("UnitreeA1.simple", p, num_envs=N, seed=3) for p in PATHS]
    for e in envs:
        e.reference_body_state
    obs = [e.reset() for e in envs]
    assert all(torch.equal(obs[0], o) for o in obs[1:])
    gen = torch.Generator().manual_seed(2)
    resets = 0
    for _ in range(8):
        act = _act(gen, N, 12)
        outs = [e.step(act) for e in envs]
        resets += int(outs[0][2].bool().sum())
        for e, o in zip(envs[1:], outs[1:]):
            assert torch.equal(outs[0][2], o[2])
            assert torch.equal(envs[0].reference_body_state, e.reference_body_state)
            assert torch.equal(envs[0].next_reference_body_state, e.next_reference_body_state)
    assert resets > 0


def test_captured_step_writes_the_registered_buffers(bundled_only):
    n, steps = 256, 8
    eager = _make("UnitreeA1.simple", num_envs=n, seed=21)
    graphed = _make("UnitreeA1.simple", num_envs=n, seed=21)
    re_, ne = eager.reference_body_state, eager.next_reference_body_state
    rg, ng = graphed.reference_body_state, graphed.next_reference_body_state    # registered before the capture
    assert torch.equal(eager.reset(), graphed.reset())
    eng = graphed._get_engine()
    static_act = torch.zeros((n, 12), device="cuda")
    warm = _make("UnitreeA1.simple", num_envs=n, seed=99)
    warm.reset()
    warm._get_engine().step(static_act)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        eng.step(static_act)
    eager._get_engine().step(torch.zeros((n, 12), device="cuda"))
    graph.replay()
    gen = torch.Generator().manual_seed(5)
    resets = 0
    for _ in range(steps):
        act = _act(gen, n, 12)
        eager.step(act)
        static_act.copy_(act)
        rg.zero_()
        ng.zero_()
        graph.replay()
        torch.cuda.synchronize()
        resets += int(eng.done.bool().sum())
        assert torch.equal(re_, rg) and torch.equal(ne, ng) and float(rg.abs().max()) > 0
    assert resets > 0


def test_two_shards_equal_one_batch(bundled_only):
    n, steps = 64, 10
    full = _make("UnitreeA1.simple", num_envs=n, seed=11)
    a = _make("UnitreeA1.simple", num_envs=n // 2, seed=11, env_id_offset=0)
    b = _make("UnitreeA1.simple", num_envs=n // 2, seed=11, env_id_offset=n // 2)
    for e in (full, a, b):
        e.next_reference_body_state
    assert torch.equal(full.reset(), torch.cat([a.reset(), b.reset()]))
    assert torch.equal(full.next_reference_body_state, torch.cat([a.next_reference_body_state, b.next_reference_body_state]))
    gen = torch.Generator().manual_seed(1)
    for _ in range(steps):
        act = _act(gen, n, 12)
        full.step(act)
        a.step(act[:n // 2].contiguous())
        b.step(act[n // 2:].contiguous())
        assert torch.equal(full.reference_body_state, torch.cat([a.reference_body_state, b.reference_body_state]))
        assert torch.equal(full.next_reference_body_state,
                           torch.cat([a.next_reference_body_state, b.next_reference_body_state]))


def test_mixed_batch_members_expose_their_own_rows(bundled_only):
    from loco_mujoco_b200.parallel import MixedBatch
    n = 48
    mb = MixedBatch([("Atlas.walk.real", n, dict(KW)), ("Talos.walk.real", n, dict(KW))], device="cuda:0", seed=3,
                    debug=True)
    solo = [make_env("Atlas.walk", num_envs=n, seed=3, env_id_offset=0, **KW),
            make_env("Talos.walk", num_envs=n, seed=3, env_id_offset=n, **KW)]
    for e in mb.envs + solo:
        e.reference_body_state
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
            assert m.reference_body_state.shape[1] == s._model.nbody
            assert torch.equal(m.reference_body_state, s.reference_body_state)
            assert torch.equal(m.next_reference_body_state, s.next_reference_body_state)


@pytest.mark.parametrize("task,kw", [("UnitreeA1.simple", dict(setup_random_rot=True)), ("HumanoidTorque.run", {}),
                                     ("Atlas.walk+arms", {})])
def test_dataset_rows_equal_pinned_resets(bundled_only, task, kw):
    """Row r of create_dataset_bodies() equals, bit for bit, next_body_state after a reset onto the row's (traj, sample)
    with angle 0 (and onto sample + 1 for next_body_states); within a trajectory next_body_states[r] is body_states[r + 1]."""
    env = _make(task, num_envs=8, seed=0, **kw)
    ds = env.create_dataset_bodies()
    body, nxt = ds["body_states"], ds["next_body_states"]
    states = env.create_dataset_device()["states"]
    n_traj, T = env.trajectories.number_of_trajectories, env.trajectories.trajectory_length
    per = T - 1
    assert body.shape == nxt.shape == (n_traj * per, env._model.nbody, 13) and len(states) == len(body)
    last = torch.arange(len(body), device="cuda") % per == per - 1
    assert torch.equal(nxt[:-1][~last[:-1]], body[1:][~last[:-1]])
    rows = torch.tensor([0, 1, per - 1, len(body) - 1, len(body) // 2, 7 * per + 3], dtype=torch.int64, device="cuda")
    rows = rows[rows < len(body)]
    cur = (rows // per) * T + rows % per
    zero = torch.zeros(len(rows), device="cuda") if kw else None
    assert torch.equal(_twin_rows(task, cur, zero, **kw), body[rows])
    assert torch.equal(_twin_rows(task, cur + 1, zero, **kw), nxt[rows])


def test_deepmimic_end_effector_term(bundled_only):
    """The usage example: DeepMimic's end-effector reward exp(-40 sum_feet |p_sim - p_ref|^2) from body_state and
    reference_body_state, with the simulated feet taken relative to the simulated root's x / y (the reference root stands
    at x = y = 0). It is 1 right after a reset and falls below 1 once random actions pull the robot off the clip."""
    n = 256
    env = _make("UnitreeA1.simple", num_envs=n, seed=5)
    m = env._model
    feet = [env.body_index(nm) for nm in m.body_names if nm.endswith("calf")]
    root = env.body_index("trunk")
    assert len(feet) == 4

    def term(body, ref):
        sim = body[:, feet, :3].clone()
        sim[..., :2] -= body[:, root, None, :2]
        return torch.exp(-40.0 * ((sim - ref[:, feet, :3]) ** 2).sum((-1, -2)))

    env.reset()
    assert bool((term(env.next_body_state, env.next_reference_body_state) == 1.0).all())
    gen = torch.Generator().manual_seed(6)
    for _ in range(10):
        _, _, done, info = env.step(_act(gen, n, 12))
    r = term(env.body_state, env.reference_body_state)
    live = ~(done | info["truncated"]).bool()
    assert bool((r[live] < 1.0).all()) and float(r[live].mean()) < 0.99 and bool(((r >= 0) & (r <= 1)).all())
