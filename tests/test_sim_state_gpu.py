"""Saved simulation states on the GPU (include/locosim.h locosim_save_state / locosim_load_state; LocoEnv.save_state /
load_state): a load followed by the same actions replays the original bit for bit on every kernel family and launch path,
with every feature that keeps per-env state turned on (time limit and end of trajectory, a parameter pool, a carry task,
setup_random_rot, the tracking reward, applied forces, body / reference / contact / dof outputs); partial loads, banks of
any size, refused rows, forks and their first reset, clamping, CUDA graphs, shards and MixedBatch members."""
import os

import numpy as np
import pytest
import torch

import sim_state_ref as ref
from full_body import make_variant
from helpers import make_env

pytestmark = pytest.mark.gpu

# launch paths of UnitreeA1 (environment variables read when an engine is created, locosim.cu setup_cfg)
PATHS = {"fused": {"LOCOSIM_RESORT": "10"}, "substeps": {"LOCOSIM_RESORT": "2"},
         "persistent": {"LOCOSIM_RESORT": "2", "LOCOSIM_PERSIST": "1"}}
# every feature that keeps per-env state: a short time limit and the end-of-trajectory limit (auto-resets inside every window)
BASE = dict(time_limit=5, truncate_at_trajectory_end=True)
# one task per kernel family: CfgEllEuler (three launch paths), CfgPyrEuler, CfgPyrRK4 (and its carry task), CfgPyrEuler29,
# CfgPyrRK4_31, CfgPyrEuler31
A1 = dict(setup_random_rot=True, reward_type="tracking")
FAMILIES = [("UnitreeA1.simple", "fused", A1), ("UnitreeA1.simple", "substeps", A1), ("UnitreeA1.simple", "persistent", A1),
            ("Talos.walk", None, dict(domain_randomization_config="domain_randomization_talos.yaml")),
            ("HumanoidTorque.run", None, dict(reward_type="tracking")), ("Atlas.carry", None, {}),
            ("UnitreeG1.walk", None, {}),
            ("Atlas.walk+arms", None, dict(domain_randomization_config="domain_randomization_atlas.yaml")),
            ("Talos.walk+arms", None, {})]
IDS = ["%s-%s" % (t, p) if p else t for t, p, _ in FAMILIES]
N = 256
OUTPUTS = ("body_state", "next_body_state", "reference_body_state", "next_reference_body_state", "contact_wrench",
           "dof_outputs", "xfrc_applied")


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


def _make(task, path=None, outputs=True, **kw):
    """env with every output registered and random applied forces on every body (set after its first reset)"""
    kw = dict(BASE, **kw)
    env = _with_env(PATHS[path] if path else {}, lambda: make_variant(task, **kw))
    _with_env(PATHS[path] if path else {}, env._get_engine)
    if outputs:
        for name in OUTPUTS:
            getattr(env, name)
    return env


def _push(env, seed):
    g = torch.Generator().manual_seed(seed)
    xf = env.xfrc_applied
    xf[:, 1:] = (torch.rand(xf[:, 1:].shape, generator=g) * 2 - 1).cuda() * 5.0


def _acts(env, k, seed, n=None):
    g = torch.Generator().manual_seed(seed)
    n = env.num_envs if n is None else n
    return [(torch.rand((n, env.info.action_space.shape[0]), generator=g) * 2 - 1).cuda() for _ in range(k)]


def _bits(x):
    return x.view(torch.int32) if x.dtype == torch.float32 else x


def _snapshot(env, step=None):
    """everything a step returns and the engine keeps, cloned"""
    eng = env._get_engine()
    out = {}
    if step is not None:
        obs, rew, done, info = step
        out.update(obs=obs, rew=rew, done=done, **info)
    q, v, w = eng.get_state()
    out.update(qpos=q, qvel=v, ws=w, cursor=eng.cursor(), rows=eng.param_rows(), stats=torch.stack(
        [x.view(torch.int32) if x.dtype == torch.float32 else x for x in eng.episode_stats()], dim=1))
    for name in OUTPUTS:
        if getattr(env, "_" + name, None) is not None:
            out[name] = getattr(env, name)
    return {k: x.clone() for k, x in out.items()}


def _run(env, acts):
    return [_snapshot(env, env.step(a)) for a in acts]


def _assert_same(a, b, rows=None, what=""):
    assert a.keys() == b.keys(), what
    for k in a:
        x, y = _bits(a[k]), _bits(b[k])
        if rows is not None:
            x, y = x[rows], y[rows]
        assert torch.equal(x, y), "%s %s differs in %d entries" % (what, k, int((x != y).sum()))


def _assert_runs_same(r1, r2, rows=None):
    assert len(r1) == len(r2)
    for j, (a, b) in enumerate(zip(r1, r2)):
        _assert_same(a, b, rows, "step %d:" % j)


def _to_k0(env, k0, seed=0):
    env.reset()
    _push(env, seed)
    for a in _acts(env, k0, seed + 100):
        obs, _, _, info = env.step(a)
    return info["next_obs"].clone()


@pytest.mark.parametrize("task,path,kw", FAMILIES, ids=IDS)
def test_load_and_replay_is_bit_identical(bundled_only, task, path, kw):
    """save at step k0, run to k1 recording everything; load the row back into the same env and replay the same actions
    (the applied forces restored in torch): every word of every step is the same, auto-resets inside the window included"""
    env = _make(task, path, num_envs=N, seed=7, **kw)
    nobs = _to_k0(env, 3)
    # (what a load writes back: the state and the rows of the state to act on next, not the last step's outputs)
    last_step = ("body_state", "reference_body_state", "contact_wrench", "dof_outputs")
    at_k0 = {k: x for k, x in _snapshot(env).items() if k not in last_step}
    xf0 = env.xfrc_applied.clone()
    state = env.save_state()
    assert state.shape == (N, env._get_engine().state_words) and state.dtype == torch.int32
    acts = _acts(env, 14, 1)
    first = _run(env, acts)
    assert sum(int((s["done"] != 0).sum() + s["truncated"].sum()) for s in first) > 0, "no reset inside the window"
    got = env.load_state(state)
    assert torch.equal(_bits(got), _bits(nobs))
    env.xfrc_applied.copy_(xf0)
    _assert_same({k: x for k, x in _snapshot(env).items() if k not in last_step}, at_k0, what="after the load:")
    _assert_runs_same(first, _run(env, acts))


@pytest.mark.parametrize("src,dst", [("fused", "persistent"), ("persistent", "substeps"), ("substeps", "fused")])
def test_replay_on_another_launch_path(bundled_only, src, dst):
    """rows saved by an engine on one launch path replay bit for bit on a fresh engine of the same task on another"""
    a = _make("UnitreeA1.simple", src, num_envs=N, seed=7, **A1)
    b = _make("UnitreeA1.simple", dst, num_envs=N, seed=7, **A1)
    _to_k0(a, 3)
    state, xf0 = a.save_state(), a.xfrc_applied.clone()
    acts = _acts(a, 12, 2)
    first = _run(a, acts)
    b.reset()
    b.load_state(state)
    b.xfrc_applied.copy_(xf0)
    _assert_runs_same(first, _run(b, acts))


@pytest.mark.parametrize("task,path,kw", [FAMILIES[2], FAMILIES[4]], ids=[IDS[2], IDS[4]])
def test_partial_load_leaves_other_envs_alone(bundled_only, task, path, kw):
    """index -1 for the odd envs: they stay bit-identical to a control engine that never loaded; the even envs replay"""
    env, ctl = _make(task, path, num_envs=N, seed=5, **kw), _make(task, path, num_envs=N, seed=5, **kw)
    for e in (env, ctl):
        _to_k0(e, 2)
    state, xf0 = env.save_state(), env.xfrc_applied.clone()
    acts = _acts(env, 10, 3)
    first = _run(env, acts)
    ctl_first = _run(ctl, acts)
    i = torch.arange(N, device="cuda", dtype=torch.int32)
    idx = torch.where(i % 2 == 0, i, -1).to(torch.int32)
    before = env._obs.clone()
    got = env.load_state(state, idx)
    assert torch.equal(_bits(got[1::2]), _bits(before[1::2]))
    env.xfrc_applied[::2] = xf0[::2]
    acts2 = _acts(env, 10, 3)
    second, ctl_second = _run(env, acts2), _run(ctl, acts2)
    _assert_runs_same(second, ctl_second, rows=slice(1, None, 2))
    _assert_runs_same(first, second, rows=slice(0, None, 2))


def test_banks_smaller_and_larger_than_the_batch(bundled_only):
    """M < n and M > n rows; indices >= M and rows with another layout tag leave the env untouched"""
    n = 64
    env = _make("UnitreeA1.simple", num_envs=n, seed=2, **A1)
    lay = env._get_engine().state_layout
    _to_k0(env, 2)
    s1 = env.save_state()
    env.step(_acts(env, 1, 9)[0])
    s2 = env.save_state()
    q0, v0 = lay["qpos"], lay["qvel"]

    def state_rows():
        q, v, _ = env._get_engine().get_state()
        return torch.cat([q, v], 1).view(torch.int32)

    i = torch.arange(n, device="cuda", dtype=torch.int32)
    small = s1[:5].clone()
    obs = env.load_state(small, (i % 5).to(torch.int32))
    assert torch.equal(state_rows(), s1[(i % 5).long(), q0[0]:v0[0] + v0[1]])
    assert torch.equal(_bits(obs), s1[(i % 5).long(), lay["obs"][0]:lay["obs"][0] + lay["obs"][1]])
    bank = torch.cat([s1, s2])
    env.load_state(bank, (i + n).to(torch.int32))
    assert torch.equal(state_rows(), s2[:, q0[0]:v0[0] + v0[1]])
    # out of range and foreign rows: untouched
    keep = env.save_state()
    foreign = s1.clone()
    foreign[:, 1] ^= 1
    env.load_state(torch.cat([s1, foreign]), torch.where(i % 2 == 0, i + n, 2 * n + i).to(torch.int32))
    assert torch.equal(env.save_state(), keep)
    obs = env.load_state(s1[:3].clone(), torch.where(i < 3, i, 3 + i).to(torch.int32))
    after = env.save_state()
    assert torch.equal(after[:3], s1[:3]) and torch.equal(after[3:], keep[3:])


FORKS = [("UnitreeA1.simple", A1), ("Talos.walk", FAMILIES[3][2]), ("Atlas.carry", {})]


@pytest.mark.parametrize("task,kw", FORKS, ids=[t for t, _ in FORKS])
def test_forks_match_until_their_own_first_reset(bundled_only, task, kw):
    """every env takes env 0's row: identical (next body and reference rows included: the angle pin) until the first reset,
    which then draws cursor, pool row and rotation from each env's own stream, as the restated draws predict"""
    n, seed = 64, 11
    env = _make(task, num_envs=n, seed=seed, **kw)
    eng = env._get_engine()
    lay = eng.state_layout
    _to_k0(env, 2)
    env.xfrc_applied.zero_()
    s = env.save_state()
    ep0 = int(s[0, lay["episode"][0]])
    obs = env.load_state(s, torch.zeros(n, dtype=torch.int32, device="cuda"))
    assert torch.equal(_bits(obs), _bits(obs[:1].expand_as(obs)))
    for name in ("next_body_state", "next_reference_body_state"):
        x = _bits(getattr(env, name))
        assert torch.equal(x, x[:1].expand_as(x)), name
    a = _acts(env, 1, 4, n=1)[0]
    for k in range(20):
        obs, _, done, info = env.step(a.expand(n, -1).contiguous())
        assert torch.equal(_bits(obs), _bits(obs[:1].expand_as(obs))), k
        for name in ("body_state", "reference_body_state", "contact_wrench", "dof_outputs"):
            x = _bits(getattr(env, name))
            assert torch.equal(x, x[:1].expand_as(x)), (k, name)
        ended = (done != 0) | info["truncated"]
        if ended.any():
            break
    assert ended.all(), "the forks did not end together"
    T, n_traj = env.trajectories.trajectory_length, env.trajectories.number_of_trajectories
    K = _pool_rows(env)
    cur, rows = eng.cursor().cpu().numpy(), eng.param_rows().cpu().numpy()
    draws = [ref.draw_reset(seed, g, ep0, n_traj, T) for g in range(n)]
    assert cur.tolist() == [t * T + sp for t, sp in draws]
    assert rows.tolist() == [ref.draw_pool_row(seed, g, ep0, K) for g in range(n)]
    assert len(set(cur.tolist())) > 1
    # the next reference rows: those of a twin reset onto the same rows, pool rows and (restated) angles
    twin = _make(task, num_envs=n, seed=seed, outputs=False, **kw)
    tw = twin._get_engine()
    nref = twin.next_reference_body_state
    c = torch.tensor(cur, dtype=torch.int32, device="cuda")
    ang = None
    if kw.get("setup_random_rot"):
        ang = torch.tensor([ref.draw_rot_angle(seed, g, ep0) for g in range(n)], dtype=torch.float32, device="cuda")
    tw.reset(traj_no=(c // T).contiguous(), step_no=(c % T).contiguous(),
             pool_row=torch.tensor(rows, dtype=torch.int32, device="cuda"), rot_angle=ang)
    assert torch.equal(_bits(env.next_reference_body_state), _bits(nref))


def _pool_rows(env):
    if env._domain_rand_config is not None:
        return len(env.domain_randomization_pool())
    return len(env._models) if (len(env._models) > 1 or len(env._model_user_features[0])) else 1


def test_carry_load_restores_the_weight(bundled_only):
    """a row loaded into an engine of another seed carries its weight (pool row and the LS_OBS_PARAM entry), and the step
    from it is the original's bit for bit"""
    a = _make("Talos.carry", num_envs=N, seed=1)
    b = _make("Talos.carry", num_envs=N, seed=2)
    _to_k0(a, 2)
    b.reset()
    assert _pool_rows(a) > 1 and not torch.equal(a._get_engine().param_rows(), b._get_engine().param_rows())
    s, xf0 = a.save_state(), a.xfrc_applied.clone()
    act = _acts(a, 1, 6)[0]
    obs_a = a.step(act)[0].clone()
    nobs = b.load_state(s)
    assert torch.equal(b._get_engine().param_rows(), s[:, 3])
    assert torch.equal(_bits(nobs), s[:, a._get_engine().state_layout["obs"][0]:][:, :nobs.shape[1]])
    b.xfrc_applied.copy_(xf0)
    assert torch.equal(_bits(b.step(act)[0]), _bits(obs_a))


def test_pool_row_and_cursor_are_clamped(bundled_only):
    """a row saved before a smaller parameter pool (or with its cursor past the table) loads in range"""
    env = _make("Talos.walk", num_envs=N, seed=3, **FAMILIES[3][2])
    eng = env._get_engine()
    lay = eng.state_layout
    _to_k0(env, 1)
    s = env.save_state()
    assert int(s[:, 3].max()) >= 2
    eng.set_param_pool(env.domain_randomization_pool()[:2])
    s[:8, lay["cursor"][0]] = 1 << 30
    s[8:16, lay["cursor"][0]] = -5
    env.load_state(s)
    assert torch.equal(eng.param_rows(), s[:, 3].clamp(0, 1))
    c = eng.cursor()
    T, n_traj = env.trajectories.trajectory_length, env.trajectories.number_of_trajectories
    assert (c[:8] == n_traj * T - 1).all() and (c[8:16] == 0).all() and torch.equal(c[16:], s[16:, lay["cursor"][0]])
    env.step(_acts(env, 1, 0)[0])
    torch.cuda.synchronize()


@pytest.mark.parametrize("task,path,kw", [FAMILIES[2], FAMILIES[4]], ids=[IDS[2], IDS[4]])
def test_graph_captured_planning_loop_equals_eager(bundled_only, task, path, kw):
    """save -> H steps -> load -> one committed step, captured once in a CUDA graph and replayed with new actions, equals
    the same calls made eagerly on a twin engine"""
    n, H = 128, 4
    envs = [_make(task, path, num_envs=n, seed=9, **kw) for _ in range(2)]
    engs = [e._get_engine() for e in envs]
    for e in envs:
        e.reset()
        _push(e, 1)
    nu = engs[0].action_dim
    bufs = [dict(acts=torch.zeros((H + 1, n, nu), device="cuda"), S=torch.empty((n, e.state_words), dtype=torch.int32,
                                                                                  device="cuda"),
                 obs=e.next_obs.clone()) for e in engs]

    def loop(eng, b):
        eng.save_state(b["obs"], out=b["S"])
        for h in range(H):
            eng.step(b["acts"][h])
        eng.load_state(b["S"], obs_out=b["obs"])
        eng.step(b["acts"][H])
        b["obs"].copy_(eng.next_obs)

    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        loop(engs[1], bufs[1])
    gen = torch.Generator().manual_seed(5)
    for r in range(6):
        a = (torch.rand((H + 1, n, nu), generator=gen) * 2 - 1).cuda()
        for b in bufs:
            b["acts"].copy_(a)
        loop(engs[0], bufs[0])
        g.replay()
        torch.cuda.synchronize()
        _assert_same(_snapshot(envs[0]), _snapshot(envs[1]), what="replay %d:" % r)
        for k in ("obs",):
            assert torch.equal(_bits(bufs[0][k]), _bits(bufs[1][k]))
        assert torch.equal(_bits(engs[0].obs), _bits(engs[1].obs)) and torch.equal(engs[0].reward.view(torch.int32),
                                                                                   engs[1].reward.view(torch.int32))


def test_shards_and_mixed_batch_members(bundled_only):
    """shards save and load their own rows, and a row moves between two shards of one task; MixedBatch members replay"""
    from loco_mujoco_b200.parallel import MixedBatch, make_sharded
    n = 64
    sh = [make_sharded("UnitreeA1.simple.real", 2 * n, rank=r, world_size=2, device="cuda:0", seed=4, debug=True,
                       **dict(BASE, **A1)) for r in range(2)]
    for e in sh:
        e.body_state
        e.reset()
    acts = _acts(sh[0], 3, 8)
    for a in acts:
        for e in sh:
            e.step(a)
    s0 = sh[0].save_state()
    first = _run(sh[0], acts)
    sh[0].load_state(s0)
    _assert_runs_same(first, _run(sh[0], acts))
    # shard 0's envs into shard 1: the same state, and the same first step (compared up to the terminal observation)
    sh[1].load_state(s0)
    assert torch.equal(sh[1].save_state(), s0)
    sh[0].load_state(s0)
    o0, r0 = (x.clone() for x in sh[0].step(acts[0])[:2])
    o1, r1 = sh[1].step(acts[0])[:2]
    assert torch.equal(_bits(o0), _bits(o1)) and torch.equal(_bits(r0), _bits(r1))

    mb = MixedBatch([("Atlas.walk.real", n, dict(BASE)), ("Talos.walk.real", n, dict(BASE))], device="cuda:0", seed=3,
                    concurrent=False, debug=True)
    mb.reset()
    acts = [_acts(e, 4, 10 + i) for i, e in enumerate(mb.envs)]
    for k in range(2):
        mb.step([a[k] for a in acts])
    # (MixedBatch.step drives the engines directly: the observation to act on next is each engine's next_obs)
    saved = [e.save_state(e.next_obs) for e in mb.engines]

    def run():
        out = []
        for k in range(4):
            mb.step([a[k] for a in acts])
            out.append([_snapshot(e) for e in mb.envs])
        return out

    first = run()
    for e, s in zip(mb.engines, saved):
        e.load_state(s)
    second = run()
    for a, b in zip(first, second):
        for x, y in zip(a, b):
            _assert_same(x, y)


def test_drop_in_mode_round_trip(bundled_only):
    """drop-in single env: the row is a device tensor and load_state returns the numpy float64 observation"""
    env = make_env("UnitreeA1.simple", seed=0)
    env.reset()
    a = np.random.RandomState(0).uniform(-1, 1, (3, 12))
    env.step(a[0])
    s = env.save_state()
    assert s.is_cuda and s.shape[0] == 1
    ref_obs = env._obs.copy()
    first = [env.step(x)[0] for x in a[1:]]
    got = env.load_state(s)
    assert isinstance(got, np.ndarray) and got.dtype == np.float64 and np.array_equal(got, ref_obs)
    second = [env.step(x)[0] for x in a[1:]]
    assert all(np.array_equal(x, y) for x, y in zip(first, second))
