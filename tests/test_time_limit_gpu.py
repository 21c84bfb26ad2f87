"""Time limit (include/locosim.h locosim_set_time_limit), GPU tier (H100). The new logic is integer bookkeeping, so the
engine, the oracle and a NumPy recount must agree flag for flag: off is off (bitwise), a recount of episode ages from the
returned done bytes, the reference model around the oracle (time_limit_ref), the reset a truncated env gets, the three launch paths, the tracking
cursor, the Gymnasium vector wrapper, sharding, the composites and a CUDA graph. One configuration per kernel family:
UnitreeA1 (elliptic cones, Euler), HumanoidTorque (RK4) and Talos with arms (the second translation unit).
The CPU tier is tests/test_time_limit.py."""
import numpy as np
import pytest

from full_body import make_variant
from helpers import oracle_env
from time_limit_ref import TimeLimitRef

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

TASKS = ["UnitreeA1.simple", "HumanoidTorque.run", "Talos.walk+arms"]
# Limits that seeded U(-1, 1) actions reach and miss in comparable numbers: random torques topple UnitreeA1 within 8 - 27 control
# steps and the humanoids within 2 - 15 (fp64 oracle, 12 episodes each)
LIMIT = {"UnitreeA1.simple": 12, "HumanoidTorque.run": 4, "Talos.walk+arms": 5}


def _rollout(env, steps, limit=None, seed=7, auto_reset=True):
    """Seeded U(-1, 1) rollout on the engine; everything it returns and its final state, as a list of tensors."""
    eng = env._get_engine()
    if limit is not None:
        eng.set_time_limit(*limit)
    out = [eng.reset().clone()]
    g = torch.Generator(device="cpu").manual_seed(seed)
    for _ in range(steps):
        act = (torch.rand((eng.n_envs, eng.action_dim), generator=g) * 2 - 1).cuda()
        out += [t.clone() for t in eng.step(act, auto_reset=auto_reset)]
    out += [t.clone() for t in eng.get_state()]
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("task", TASKS)
def test_off_is_off_and_an_unreached_limit_changes_nothing(bundled_only, task):
    n, steps = 512, 60
    never = _rollout(make_variant(task, num_envs=n, seed=5), steps)
    done = torch.stack(never[3:-3:4])
    assert set(done.unique().tolist()) <= {0, 1} and int(done.sum()) > 0, "expected some terminations and no other byte"
    for limit in ((0, False), (10 ** 6, False)):
        got = _rollout(make_variant(task, num_envs=n, seed=5), steps, limit=limit)
        for i, (a, b) in enumerate(zip(never, got)):
            assert torch.equal(a, b), "set_time_limit%s changes output %d" % (limit, i)


@pytest.mark.parametrize("task", TASKS)
def test_truncation_and_episode_statistics_against_a_recount(bundled_only, task):
    """From the returned done bytes alone: episode ages reproduce every truncated bit, no episode exceeds the limit, the reset
    counter is the number of finished episodes, and the engine's episode length / return are the recount of the returned
    rewards (fp32, summed in step order: exactly)."""
    n, steps, H = 512, 120, LIMIT[task]
    env = make_variant(task, num_envs=n, seed=5)
    eng = env._get_engine()
    eng.set_time_limit(H, False)
    eng.reset()
    age, ret = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.float32)
    finished = np.zeros(n, dtype=np.int64)
    last_len, last_ret = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.float32)
    n_trunc = n_abs = 0
    g = torch.Generator(device="cpu").manual_seed(7)
    for k in range(steps):
        act = (torch.rand((n, eng.action_dim), generator=g) * 2 - 1).cuda()
        _, rew, done, _ = eng.step(act)
        stats = [t.cpu().numpy() for t in eng.episode_stats()]
        rew, done = rew.cpu().numpy(), done.cpu().numpy()
        assert set(np.unique(done).tolist()) <= {0, 1, 2}
        age += 1
        ret = (ret + rew).astype(np.float32)
        absorbing, truncated = (done & 1) != 0, (done & 2) != 0
        assert np.array_equal(truncated, (age == H) & ~absorbing), "step %d" % k
        assert age.max() <= H
        fin = done != 0
        last_len[fin], last_ret[fin] = age[fin], ret[fin]
        finished += fin
        age[fin], ret[fin] = 0, 0
        assert np.array_equal(stats[0], age) and np.array_equal(stats[1], ret), "running pair, step %d" % k
        assert np.array_equal(stats[2], last_len) and np.array_equal(stats[3], last_ret), "finished pair, step %d" % k
        n_trunc += int(truncated.sum())
        n_abs += int(absorbing.sum())
    assert n_trunc > 0 and n_abs > 0, (n_trunc, n_abs)
    cnt = eng.counters().cpu().numpy()
    assert np.array_equal(cnt[:, 1], finished + 1) and (cnt[:, 0] == steps).all()


def _near_threshold(env, obs, eps=1e-3):
    """the rule of test_gpu_parity for a done flag that differs between fp32 and fp64"""
    for key, lo, hi in env._has_fallen_terms():
        v = obs[env.get_obs_idx(key)[0]]
        if abs(v - lo) < eps or abs(v - hi) < eps:
            return True
    return False


@pytest.mark.parametrize("task", TASKS)
def test_flags_match_the_oracle(oracle, bundled_only, task):
    """64 envs pinned to reset rows up to 15 samples before the end of their trajectory, both limits on, no auto-reset (the
    flags then repeat until a reset). Bit 1 has no tolerance; bit 0 has the existing one (near a threshold, or after the fp32
    rollout has left the fp64 one), and where bit 0 differs bit 1 is decided by it (absorbing wins)."""
    n, steps, H = 64, 12, 5
    env = make_variant(task, num_envs=n, seed=5, warps_per_block=8)
    eng = env._get_engine()
    eng.set_time_limit(H, True)
    T = env.trajectories.trajectory_length
    tr = (np.arange(n) % env.trajectories.number_of_trajectories).astype(np.int32)
    st = (T - 1 - (np.arange(n) % 16)).astype(np.int32)
    obs0 = eng.reset(traj_no=torch.tensor(tr, device=eng.device), step_no=torch.tensor(st, device=eng.device)).cpu().numpy()
    oes = [TimeLimitRef(oracle_env(oracle, env), env) for _ in range(n)]
    for i, oe in enumerate(oes):
        oe.set_time_limit(H, True)
        assert np.abs(oe.reset_to(tr[i], st[i]) - obs0[i]).max() < 1e-5
    rng = np.random.RandomState(0)
    same = np.ones(n, dtype=bool)            # the fp32 rollout still follows the fp64 one, and neither has fallen
    compared = n_trunc = 0
    for k in range(steps):
        act = (0.3 * rng.uniform(-1, 1, (n, eng.action_dim))).astype(np.float32)
        obs, _, done, _ = eng.step(torch.tensor(act, device=eng.device), auto_reset=False)
        obs, done = obs.cpu().numpy(), done.cpu().numpy()
        cur = eng.cursor().cpu().numpy()
        for i, oe in enumerate(oes):
            o, _, ab, trunc = oe.step_ex(act[i].astype(np.float64))
            want_limit = k + 1 >= min(H, max(T - 1 - st[i], 1))
            assert oe.cursor() == cur[i] == tr[i] * T + min(st[i] + k + 1, T - 1)
            if bool(done[i] & 1) != ab:
                assert not same[i] or _near_threshold(env, o), "absorbing flag differs away from the threshold"
                same[i] = False
                assert bool(done[i] & 2) == (want_limit and not done[i] & 1)
                continue
            assert bool(done[i] & 2) == trunc == (want_limit and not ab), (task, k, i, done[i], ab, trunc)
            compared += 1
            n_trunc += int(trunc)
            if ab or not np.allclose(obs[i], o, rtol=2e-3 * (k + 1), atol=2e-3 * (k + 1)):
                same[i] = False
    for oe in oes:
        oe.close()
    assert compared > n * steps // 4 and n_trunc > 0, (compared, n_trunc)


def test_a_truncated_env_gets_the_reset_of_its_next_episode(bundled_only):
    """auto_reset: `obs` is the stepped state's observation (what an engine without a limit returns for the same step),
    `next_obs` the reset observation of the env's NEXT episode number: the second draw of the counter-based stream, and
    bit for bit what locosim_reset_rows writes for that (trajectory, sample, pool row)."""
    n, H = 256, 9
    envs = [make_variant("UnitreeA1.simple", num_envs=n, seed=5) for _ in range(4)]
    limited, free, drawn, pinned = (e._get_engine() for e in envs)
    limited.set_time_limit(H, False)
    assert torch.equal(limited.reset(), free.reset())
    g = torch.Generator(device="cpu").manual_seed(3)
    fresh = torch.ones(n, dtype=torch.bool, device="cuda")          # still in the first episode
    for k in range(H):
        act = (torch.rand((n, 12), generator=g) * 2 - 1).cuda()
        obs, rew, done, nxt = limited.step(act)
        obs_f, rew_f, done_f, _ = free.step(act)
        assert torch.equal(obs[fresh], obs_f[fresh]) and torch.equal(rew[fresh], rew_f[fresh])
        assert torch.equal(done[fresh] & 1, done_f[fresh])
        if k < H - 1:
            fresh &= done == 0
    trunc = fresh & (done == 2)
    assert int(trunc.sum()) > 0 and torch.equal(fresh & (done != 1), trunc)
    assert not torch.equal(obs[trunc], nxt[trunc])
    drawn.reset()
    second = drawn.reset().clone()                                   # reset number 1 of every env: the draw of episode 1
    assert torch.equal(nxt[trunc], second[trunc])
    assert torch.equal(limited.cursor()[trunc], drawn.cursor()[trunc])
    assert torch.equal(limited.counters()[trunc, 1], torch.full((int(trunc.sum()),), 2, dtype=torch.int32, device="cuda"))
    T = envs[0].trajectories.trajectory_length
    cur = limited.cursor()
    again = pinned.reset(traj_no=(cur // T).int().contiguous(), step_no=(cur % T).int().contiguous(),
                         pool_row=limited.param_rows())
    assert torch.equal(nxt[trunc], again[trunc])
    ln, ret, last_ln, _ = limited.episode_stats()
    assert int(ln[trunc].abs().sum()) == 0 and float(ret[trunc].abs().sum()) == 0.0 and bool((last_ln[trunc] == H).all())


PATHS = [({"LOCOSIM_PERSIST": "1", "LOCOSIM_RESORT": "2"}, 1),      # the persistent kernel (UnitreeA1's default at 4096 envs)
         ({"LOCOSIM_PERSIST": "0", "LOCOSIM_RESORT": "2"}, 5),      # separate sub-step launches
         ({"LOCOSIM_RESORT": "10"}, 2)]                             # the fused kernel (+ the regrouping kernel)


def test_the_three_launch_paths_agree_with_a_limit_on(bundled_only, monkeypatch):
    n, steps, H = 2000, 40, 9                                        # (9: not a multiple of the chunk length)
    runs = []
    for knobs, launches in PATHS:
        for k, v in knobs.items():
            monkeypatch.setenv(k, v)
        env = make_variant("UnitreeA1.simple", num_envs=n, seed=5, warps_per_block=15)
        assert env._get_engine().kernels_per_step == launches, knobs
        out = _rollout(env, steps, limit=(H, True))
        eng = env._get_engine()
        out += [t.clone() for t in eng.episode_stats()] + [eng.cursor().clone(), eng.counters()[:, 0:5].clone()]
        runs.append(out)
        for k in knobs:
            monkeypatch.delenv(k)
    done = torch.stack(runs[0][3:-9:4])
    assert int((done == 2).sum()) > 0 and int((done == 1).sum()) > 0
    for (knobs, _), got in zip(PATHS[1:], runs[1:]):
        for i, (a, b) in enumerate(zip(runs[0], got)):
            assert torch.equal(a, b), "%s differs from the persistent kernel in output %d" % (knobs, i)


def test_tracking_reward_never_rewards_a_row_twice(bundled_only):
    """reward_type="tracking" with end_of_trajectory: within an episode the cursor moves by exactly one row per step, and the
    step that puts it on the trajectory's last row ends the episode (without the option it would rest there)."""
    n, steps = 256, 130
    env = make_variant("UnitreeA1.simple", num_envs=n, seed=5, reward_type="tracking")
    eng = env._get_engine()
    eng.set_time_limit(0, True)
    T = env.trajectories.trajectory_length
    eng.reset()
    prev = eng.cursor().cpu().numpy()
    age = np.zeros(n, dtype=np.int64)
    g = torch.Generator(device="cpu").manual_seed(7)
    n_trunc = 0
    for k in range(steps):
        # (small actions: long episodes, so that many reach the end of their clip)
        act = 0.1 * (torch.rand((n, 12), generator=g) * 2 - 1).cuda()
        _, rew, done, _ = eng.step(act)
        done, cur = done.cpu().numpy(), eng.cursor().cpu().numpy()
        age += 1
        live, trunc = done == 0, done == 2
        assert np.array_equal(cur[live], prev[live] + 1) and (cur[live] % T < T - 1).all(), "step %d" % k
        assert (prev[trunc] % T >= T - 2).all() and (age[trunc & (prev % T == T - 1)] == 1).all()
        assert (age <= T - 1).all()
        assert bool(((rew >= 0) & (rew <= 1)).all())
        age[~live] = 0
        n_trunc += int(trunc.sum())
        prev = cur
    assert n_trunc > 0


def test_vector_gymnasium_wrapper_reports_truncation(bundled_only):
    from loco_mujoco_b200 import VectorGymnasiumWrapper
    n, H = 64, 10
    venv = VectorGymnasiumWrapper("UnitreeA1.simple.real", num_envs=n, debug=True, seed=3, time_limit=H)
    eng = venv.unwrapped._get_engine()
    obs, _ = venv.reset()
    g = torch.Generator(device="cpu").manual_seed(1)
    n_trunc = n_term = 0
    for _ in range(50):
        obs, rew, term, trunc, info = venv.step((torch.rand((n, 12), generator=g) * 2 - 1).cuda())
        assert torch.equal(term, (eng.done & 1) != 0) and torch.equal(trunc, (eng.done & 2) != 0)
        _, _, last_len, last_ret = eng.episode_stats()
        assert torch.equal(info["episode"]["l"], last_len) and torch.equal(info["episode"]["r"], last_ret)
        assert torch.equal(info["_episode"], term | trunc)
        assert bool((info["episode"]["l"][trunc] == H).all()) and bool((info["episode"]["l"][term] <= H).all())
        keep = ~(term | trunc)
        assert torch.equal(obs[keep], info["final_obs"][keep])
        assert not torch.equal(obs[trunc], info["final_obs"][trunc]) or not bool(trunc.any())
        n_trunc += int(trunc.sum())
        n_term += int(term.sum())
    assert n_trunc > 0 and n_term > 0


def test_sharded_envs_equal_single_batch_with_a_limit_on(bundled_only):
    n, steps, kw = 64, 40, dict(seed=11, time_limit=10, truncate_at_trajectory_end=True)
    full = make_variant("UnitreeA1.simple", num_envs=n, **kw)
    a = make_variant("UnitreeA1.simple", num_envs=n // 2, env_id_offset=0, **kw)
    b = make_variant("UnitreeA1.simple", num_envs=n // 2, env_id_offset=n // 2, **kw)
    assert torch.equal(full.reset(), torch.cat([a.reset(), b.reset()]))
    g = torch.Generator(device="cpu").manual_seed(1)
    n_trunc = 0
    for _ in range(steps):
        act = (torch.rand((n, 12), generator=g) * 2 - 1).cuda()
        of, rf, df, info_f = full.step(act)
        oa, ra, da, info_a = a.step(act[:n // 2].contiguous())
        ob, rb, db, info_b = b.step(act[n // 2:].contiguous())
        assert torch.equal(of, torch.cat([oa, ob])) and torch.equal(rf, torch.cat([ra, rb])) and torch.equal(df, torch.cat([da, db]))
        assert sorted(info_f) == ["episode_length", "episode_return", "next_obs", "truncated"]
        for key in info_f:
            assert torch.equal(info_f[key], torch.cat([info_a[key], info_b[key]])), key
        n_trunc += int(info_f["truncated"].sum())
    assert n_trunc > 0


def test_composites_hand_the_limit_to_their_members(bundled_only):
    from loco_mujoco_b200.engine import split_done
    from loco_mujoco_b200.parallel import MixedBatch
    H = 6
    # (concurrent: the calibration rebuilds the members' engines, which must come back with the limit set)
    mb = MixedBatch([("Atlas.walk.real", 48, {}), ("Talos.walk.real", 48, {})], device="cuda:0", seed=3, debug=True, time_limit=H)
    mb.reset()
    ages = [torch.zeros(48, dtype=torch.int64, device="cuda") for _ in mb.engines]
    n_trunc = 0
    for k in range(2 * H):
        out = mb.step([torch.zeros((48, e.action_dim), device="cuda") for e in mb.engines])
        torch.cuda.synchronize()
        for age, o in zip(ages, out):
            absorbing, truncated = split_done(o[2])
            age += 1
            assert torch.equal(truncated, (age == H) & ~absorbing)
            age[absorbing | truncated] = 0
            n_trunc += int(truncated.sum())
    assert n_trunc > 0

    env = make_variant("HumanoidTorque4Ages.walk.all", num_envs=16, seed=3, time_limit=H)
    env.reset()
    age = torch.zeros(16, dtype=torch.int64, device="cuda")
    n_trunc = 0
    for k in range(2 * H):
        _, _, done, info = env.step(torch.zeros((16, env.info.action_space.shape[0]), device="cuda"))
        age += 1
        assert torch.equal(info["truncated"], (age == H) & ~done)
        fin = done | info["truncated"]
        assert torch.equal(info["episode_length"][fin], age[fin].int())
        age[fin] = 0
        n_trunc += int(info["truncated"].sum())
    assert n_trunc > 0


def test_step_with_a_limit_is_cuda_graph_capturable(bundled_only):
    """One capture of a step with a limit on, replayed 30 times, equals 30 eager steps (the limit is a kernel argument, the
    episode statistics live in device memory: nothing of it is host state)."""
    n, steps, H = 256, 30, 7
    eager = make_variant("UnitreeA1.simple", num_envs=n, seed=21, time_limit=H)
    graphed = make_variant("UnitreeA1.simple", num_envs=n, seed=21, time_limit=H)
    assert torch.equal(eager.reset(), graphed.reset())
    eng = graphed._get_engine()
    static_act = torch.zeros((n, 12), device="cuda")
    warm = make_variant("UnitreeA1.simple", num_envs=n, seed=99)     # loads the kernels outside the capture (lazy module load)
    warm.reset()
    warm._get_engine().step(static_act)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        eng.step(static_act)
    gen = torch.Generator(device="cpu").manual_seed(5)
    n_trunc = 0
    for _ in range(steps):
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        obs, rew, done, info = eager.step(act)
        static_act.copy_(act)
        graph.replay()
        assert torch.equal(obs, eng.obs) and torch.equal(rew, eng.reward) and torch.equal(info["next_obs"], eng.next_obs)
        assert torch.equal(done.to(torch.uint8) + 2 * info["truncated"].to(torch.uint8), eng.done)
        n_trunc += int(info["truncated"].sum())
    assert n_trunc > 0
    for a, b in zip(eager._get_engine().episode_stats(), eng.episode_stats()):
        assert torch.equal(a, b)
