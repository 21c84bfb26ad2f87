"""
Multi-GPU plumbing: environments are independent (SURVEY.md 8(e)), so the env axis is sharded across ranks, one process
per GPU (`torch.distributed`, NCCL over NVLink between GPUs, gloo in the CPU tests). There is no collective on the
data path of `step()`; the only (optional) exchange is an all-gather of the rollout buffer for consumers that want the
global batch on every rank.
"""
import torch
import torch.distributed as dist


def shard_range(n_total, world_size, rank):
    """Contiguous, balanced [offset, offset+count) slice of the global env axis owned by `rank`."""
    base, rem = divmod(int(n_total), int(world_size))
    count = base + (1 if rank < rem else 0)
    offset = rank * base + min(rank, rem)
    return offset, count


def make_sharded(task_id, n_total, rank=None, world_size=None, device=None, seed=0, **kwargs):
    """LocoEnv for this rank's shard; `env_id_offset` keeps every env's random stream identical to the 1-GPU run.
    Its `xfrc_applied` / `qfrc_applied`, `body_state` / `next_body_state`, `reference_body_state` /
    `next_reference_body_state`, `contact_wrench`, `dof_outputs` and `contacts`, what `inverse_dynamics(qacc)` and
    `forward_dynamics(action)` take and return and what `dynamics_terms()` returns hold the rows of this shard's envs only
    (global env offset + i is row i). So does `save_state()`; its rows load into any shard of the same task. So do
    `ray_cast(...)` and `camera(...)`, and `render(env=i)` draws this shard's env i."""
    from . import LocoEnv
    rank = dist.get_rank() if rank is None else rank
    world_size = dist.get_world_size() if world_size is None else world_size
    offset, count = shard_range(n_total, world_size, rank)
    device = device or ("cuda:%d" % (rank % max(1, torch.cuda.device_count())))
    return LocoEnv.make(task_id, num_envs=count, device=device, seed=seed, env_id_offset=offset, **kwargs)


def gather_rollout(obs, reward, done, group=None):
    """all-gather of the per-rank rollout buffer -> (obs[N_total, D], reward[N_total], done[N_total]) in global env
    order. Shards may differ by one env (shard_range), so shorter shards are padded for the collective."""
    world = dist.get_world_size(group)
    n = torch.tensor([obs.shape[0]], device=obs.device, dtype=torch.int64)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n, group=group)
    sizes = [int(s.item()) for s in sizes]
    nmax = max(sizes)
    buf = torch.zeros((nmax, obs.shape[1] + 2), device=obs.device, dtype=obs.dtype)
    buf[:obs.shape[0], :-2] = obs
    buf[:obs.shape[0], -2] = reward
    buf[:obs.shape[0], -1] = done.to(obs.dtype)
    out = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(out, buf, group=group)
    cat = torch.cat([o[:s] for o, s in zip(out, sizes)], dim=0)
    return cat[:, :-2], cat[:, -2], cat[:, -1] > 0.5


class RolloutGather:
    """The one collective the path has (SURVEY.md 8(e)): an all-gather of the rollout buffer for consumers that want the
    global batch on every rank. Per-step records are latency bound (4096 envs x 153 B = 0.6 MB), so the engine writes
    `chunk` consecutive steps straight into one time-major buffer [chunk, record_bytes] (no staging copies: `slot(t)` is
    handed to `CudaEngine.step(packed=...)`), and ONE `all_gather_into_tensor` per chunk runs on a side stream while
    the next chunk is being simulated into the second buffer (double buffering, event ordered, no host sync).

        g = RolloutGather(record_bytes, chunk, device)
        for k in range(steps):
            eng.step(actions[k], packed=g.slot())      # writes step k of the current chunk
            g.advance()                                 # after `chunk` steps: launches the gather of the full buffer
        out = g.finish()                                # [world, chunk, record_bytes] of the last complete chunk
    """

    def __init__(self, record_bytes, chunk, device, group=None):
        self.group, self.chunk, self.record_bytes = group, int(chunk), int(record_bytes)
        self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        pad = (-self.record_bytes) % 16                       # keep every time slot 16-byte aligned
        self.stride = self.record_bytes + pad
        self.local = [torch.zeros((self.chunk, self.stride), dtype=torch.uint8, device=device) for _ in range(2)]
        self.glob = [torch.zeros((self.world, self.chunk, self.stride), dtype=torch.uint8, device=device) for _ in range(2)]
        on_gpu = torch.device(device).type == "cuda"
        self.side = torch.cuda.Stream(device=device) if on_gpu else None
        self.filled = [torch.cuda.Event() for _ in range(2)] if on_gpu else None     # chunk written (compute stream)
        self.gathered = [torch.cuda.Event() for _ in range(2)] if on_gpu else None   # gather done (side stream)
        self.cur, self.t, self.n_gathers, self.last = 0, 0, 0, None
        self._pending = [False, False]

    def slot(self):
        return self.local[self.cur][self.t, :self.record_bytes]

    def bytes_received_per_chunk(self):
        return (self.world - 1) * self.chunk * self.stride

    def advance(self):
        self.t += 1
        if self.t < self.chunk:
            return False
        b = self.cur
        if self.side is not None:
            self.filled[b].record()                            # on the caller's (compute) stream
            with torch.cuda.stream(self.side):
                self.side.wait_event(self.filled[b])
                self._collective(b)
                self.gathered[b].record()
        else:
            self._collective(b)
        self._pending[b] = True
        self.last, self.n_gathers = b, self.n_gathers + 1
        self.cur, self.t = 1 - b, 0
        if self.side is not None and self._pending[self.cur]:  # the buffer about to be rewritten must have been sent
            torch.cuda.current_stream().wait_event(self.gathered[self.cur])
            self._pending[self.cur] = False
        return True

    def _collective(self, b):
        if self.world > 1:
            dist.all_gather_into_tensor(self.glob[b].view(-1), self.local[b].view(-1), group=self.group)
        else:
            self.glob[b][0].copy_(self.local[b])

    def finish(self):
        """Make the compute stream wait for every outstanding gather; returns the last gathered chunk (or None)."""
        if self.side is not None:
            for b in range(2):
                if self._pending[b]:
                    torch.cuda.current_stream().wait_event(self.gathered[b])
                    self._pending[b] = False
        return None if self.last is None else self.glob[self.last][:, :, :self.record_bytes]


class MixedBatch:
    """Heterogeneous batch on ONE GPU (BASELINE config 4: Atlas.walk + Talos.walk): the robots differ in nv, observation
    size and integrator, i.e. in the step-kernel instantiation, so every member is its own homogeneous engine.

        mb = MixedBatch([("Atlas.walk.real", 1024, {...}), ("Talos.walk.real", 1024, {...})], device="cuda:0", seed=0)
        obs = mb.reset();  results = mb.step([a_atlas, a_talos])      # lists, one entry per member

    Scheduling (results do not depend on it). A sub-batch that cannot give every SM a full block is spread by its engine
    over all SMs in smaller blocks (1024 envs on 132 SMs -> 128 blocks of 8). The members' kernels run on one stream each so
    that the light member's blocks fill the SMs the heavy member's early-finishing blocks free; which kernel the block
    scheduler places FIRST decides between a fast mode (Atlas' blocks first, config 4) and a slow one (Talos' first, back to
    back on one stream, or full blocks for both), so the members are timed alone once
    (`balance=True`) and the slowest one gets the high-priority stream: its blocks are dispatched first whenever both
    kernels have blocks pending; the lighter members run in full blocks (two spread kernels sharing every SM still hit the slow
    mode in 1 of 4 runs, spread + full blocks in 0 of 8).

    `time_limit` / `truncate_at_trajectory_end` (LocoEnv keyword arguments, for all members through `**common` or per member)
    reach every member's engine. `step` returns the engines' own tuples, so `done` is the byte of include/locosim.h:
    `engine.split_done(done)` gives the absorbing and truncated masks, `engines[i].episode_stats()` the episode numbers.
    Applied forces are per member: `envs[i].xfrc_applied` / `envs[i].qfrc_applied` / `envs[i].body_index(name)`.
    So are body outputs: `envs[i].body_state` / `envs[i].next_body_state`, reference outputs:
    `envs[i].reference_body_state` / `envs[i].next_reference_body_state`, contact outputs: `envs[i].contact_wrench`, dof
    outputs: `envs[i].dof_outputs`, the contact list: `envs[i].contacts`, inverse dynamics: `envs[i].inverse_dynamics(qacc)` / `envs[i].dof_index(joint)`,
    dynamics terms: `envs[i].dynamics_terms(...)`, forward dynamics: `envs[i].forward_dynamics(action, ...)`, ray casting:
    `envs[i].ray_cast(...)` / `envs[i].camera(...)` / `envs[i].render(env=k)`, and saved
    states: `engines[i].save_state(engines[i].next_obs)` / `engines[i].load_state(rows, index, engines[i].next_obs)` (`step`
    drives the engines, so a member's observation to act on next is its engine's `next_obs`).
    """

    def __init__(self, members, device="cuda:0", seed=0, env_id_offset=0, concurrent=True, balance=True, stagger_us=40.0, **common):
        from . import LocoEnv
        self.device = torch.device(device)
        self.stagger_cycles = int(stagger_us * 2000) if (concurrent and balance) else 0      # (~2 GHz SM clock)
        self.envs, off = [], int(env_id_offset)
        for task_id, n, kw in members:
            kw = dict(common, **(kw or {}))
            self.envs.append(LocoEnv.make(task_id, num_envs=int(n), device=str(self.device), seed=seed, env_id_offset=off, **kw))
            off += int(n)
        order = list(range(len(self.envs)))
        if concurrent and balance and len(self.envs) > 1:
            cost = self._calibrate()
            order = sorted(order, key=lambda i: -cost[i])
        self.engines = [e._get_engine() for e in self.envs]
        self.launch_order = order                      # heaviest first
        self.streams = None
        if concurrent:
            lo, hi = 0, -1                               # torch: a lower number is a higher priority
            self.streams = [torch.cuda.Stream(device=self.device, priority=hi if (i == order[0] and len(order) > 1) else lo)
                            for i in range(len(self.envs))]
        self.num_envs = sum(e.num_envs for e in self.envs)

    def _calibrate(self, steps=6):
        """ms per step of every member alone (random actions); the engines are rebuilt afterwards so that the calibration does
        not shift the envs' counter-based random streams."""
        cost = []
        for env in self.envs:
            eng = env._get_engine()
            eng.reset()
            a = torch.rand((eng.n_envs, eng.action_dim), device=self.device) * 2 - 1
            for _ in range(3):
                eng.step(a, auto_reset=True)
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(steps):
                eng.step(a, auto_reset=True)
            t1.record()
            torch.cuda.synchronize(self.device)
            cost.append(t0.elapsed_time(t1) / steps)
        slowest = max(range(len(cost)), key=lambda i: cost[i])
        for i, env in enumerate(self.envs):
            # every engine is dropped and rebuilt fresh on next use. Geometry: the slowest member keeps the engine's choice (spread),
            # the lighter ones run in FULL blocks (-1) unless the caller fixed a geometry: two spread kernels sharing every SM
            # still fell into the slow mode now and then (1 of 4 runs), spread + full blocks never did (0 of 8).
            wpb = getattr(env, "_warps_per_block", None)
            env.set_launch_geometry(wpb if (wpb is not None or i == slowest) else -1)
        self.calibration_ms = cost
        return cost

    def reset(self):
        return [e.reset() for e in self.envs]

    def step(self, actions, packed=None):
        """actions: one [n_i, nu_i] tensor per member. All members are enqueued before anything is awaited."""
        if self.streams is None:
            return [eng.step(actions[i], auto_reset=True, packed=None if packed is None else packed[i])
                    for i, eng in enumerate(self.engines)]
        cur = torch.cuda.current_stream(self.device)
        ready = torch.cuda.Event()
        ready.record(cur)
        out = []
        out = [None] * len(self.engines)
        for k, i in enumerate(self.launch_order):
            eng, st = self.engines[i], self.streams[i]
            st.wait_event(ready)
            with torch.cuda.stream(st):
                if k > 0 and self.stagger_cycles > 0:
                    # the lighter members start a few tens of microseconds after the heaviest one, so that ITS blocks are on the
                    # SMs first (its one-block regrouping kernel has to finish before its step kernel can start)
                    torch.cuda._sleep(self.stagger_cycles)
                out[i] = eng.step(actions[i], auto_reset=True, packed=None if packed is None else packed[i])
        for st in self.streams:
            cur.wait_stream(st)
        return out


def aggregate_throughput(local_units, local_seconds, device=None, group=None):
    """Whole-job throughput = units of all ranks / max-over-ranks time (the bench contract)."""
    t = torch.tensor([float(local_seconds)], dtype=torch.float64, device=device)
    u = torch.tensor([float(local_units)], dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
        dist.all_reduce(u, op=dist.ReduceOp.SUM, group=group)
    return float(u.item()) / float(t.item()), float(t.item())
