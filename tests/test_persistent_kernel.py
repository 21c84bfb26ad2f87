"""Persistent sub-step kernel (LOCOSIM_PERSIST, loco_mujoco_b200/csrc/locosim.cu persist_kernel): the control step runs as
ONE launch in which blocks pop groups of envs for chunks of sub-steps from a device-side queue of key buckets. Which block
runs which env and chunk, and in which order, is pure scheduling, so the results must be the fused kernel's bits.

CPU tier: (i) a serial model of the queue (chunks of 1, 2, 3 sub-steps, groups popped in a seeded random order with random
sizes, the working set poisoned between chunks) reproduces the uninterrupted serial build bit for bit and steps every env
through every chunk exactly once, in order; (ii) the kernel compiles for sm_90a within the sub-step kernel's registers and
stack. GPU tier: bitwise identity with the fused kernel over 50 auto-resetting steps, and CUDA-graph replay."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from helpers import ROOT, make_env
from test_substep_launches import _ptxas_report


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class _QueueModel:
    """Serial model of persist_kernel's queue: per chunk 128 key buckets; a pop takes up to `want` envs of the lowest chunk
    whose ready envs reach min(pool * want, what the chunk has left), highest keys first; groups in flight finish in random
    order and publish their envs into the next chunk (the last chunk into chunk 0 of the next step)."""

    def __init__(self, n_envs, nch, rng, pool=2):
        self.n, self.nch, self.rng, self.pool = n_envs, nch, rng, pool
        self.buckets = [[[] for _ in range(128)] for _ in range(nch)]
        self.buckets[0][0] = list(range(n_envs))
        self.taken = [0] * nch
        self.next0 = []                  # (env, key) published by the last chunk: chunk 0 of the next step

    def publish(self, c, env, key):
        self.buckets[c][min(max(key, 0), 127)].append(env)

    def pop(self, want):
        for c in range(self.nch):
            left = self.n - self.taken[c]
            ready = sum(len(b) for b in self.buckets[c])
            if left == 0 or ready == 0 or ready < min(self.pool * want, left):
                continue
            got = []
            for b in reversed(self.buckets[c]):
                while b and len(got) < want:
                    got.append(b.pop(0))
            self.taken[c] += len(got)
            return c, got
        return None


@pytest.mark.parametrize("task,kw", [("UnitreeA1.simple", {}), ("UnitreeA1.simple", {"use_foot_forces": True}),
                                     ("Talos.walk", {})])
def test_queue_order_reproduces_the_uninterrupted_step(emu, bundled_only, task, kw):
    from loco_mujoco_b200 import modelpack
    for f in ("emu_poison", "emu_iter"):
        getattr(emu, f).argtypes = [ctypes.c_void_p]
    emu.emu_poison.restype = None
    emu.emu_set_grf.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    emu.emu_get_grf.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    env = make_env(task, **kw)
    m, spec = env._model, env.task_spec()
    ints, reals = modelpack.pack(m)
    nsub, nv, n_envs = spec.n_substeps, m.nq, 6
    grp = np.ascontiguousarray(spec.grf_group, dtype=np.int32)
    table = spec.table.reshape(-1, spec.table.shape[-1])
    for chunk in (1, 2, 3):
        rng = np.random.default_rng(chunk)
        nch = -(-nsub // chunk)
        ref = [emu.emu_create(_p(ints), len(ints), _p(reals), len(reals)) for _ in range(n_envs)]
        got = [emu.emu_create(_p(ints), len(ints), _p(reals), len(reals)) for _ in range(n_envs)]
        for s in ref + got:
            assert s
            if spec.n_grf:
                emu.emu_set_grf(s, _p(grp), len(grp), spec.n_grf)
        for i in range(n_envs):
            row = table[rng.integers(len(table))]
            for s in (ref[i], got[i]):
                emu.emu_reset(s, _p(np.ascontiguousarray(row[:nv])), _p(np.ascontiguousarray(row[nv:2 * nv])))
        q = _QueueModel(n_envs, nch, rng)
        for step in range(6):
            ctrl = np.zeros((n_envs, m.nu))
            ctrl[:, spec.act_idx] = rng.uniform(-1, 1, (n_envs, m.nu)) * spec.act_delta + spec.act_mean
            for i in range(n_envs):
                emu.emu_step(ref[i], _p(np.ascontiguousarray(ctrl[i])), nsub)
            done_chunks = np.zeros(n_envs, dtype=int)
            flight = []
            while True:
                popped = q.pop(int(rng.integers(1, 5))) if rng.random() < 0.5 or not flight else None
                if popped is not None:
                    c, envs = popped
                    assert envs and all(done_chunks[e] == c for e in envs), (c, envs, done_chunks)
                    flight.append(popped)
                    continue
                if not flight:
                    break
                c, envs = flight.pop(int(rng.integers(len(flight))))
                for e in envs:
                    iters = 0
                    for _ in range(c * chunk, min((c + 1) * chunk, nsub)):
                        emu.emu_step(got[e], _p(np.ascontiguousarray(ctrl[e])), 1)
                        iters += emu.emu_iter(got[e])
                    emu.emu_poison(got[e])
                    done_chunks[e] += 1
                    if c + 1 < nch:
                        q.publish(c + 1, e, iters)
                    else:
                        q.next0.append((e, iters))
            assert (done_chunks == nch).all() and q.taken == [n_envs] * nch, (done_chunks, q.taken)
            # the next step starts from the keys of the last chunk
            nxt = _QueueModel(n_envs, nch, rng)
            nxt.buckets[0][0] = []
            for e, k in q.next0:
                nxt.publish(0, e, k)
            q = nxt
            a, b, ga, gb = np.zeros(nv), np.zeros(nv), np.zeros(12), np.zeros(12)
            for i in range(n_envs):
                emu.emu_get_state(ref[i], _p(a), _p(b))
                qa, va = a.copy(), b.copy()
                emu.emu_get_state(got[i], _p(a), _p(b))
                emu.emu_get_grf(ref[i], _p(ga), 1)
                emu.emu_get_grf(got[i], _p(gb), 1)
                assert np.array_equal(qa, a) and np.array_equal(va, b), "chunk %d step %d env %d" % (chunk, step, i)
                assert np.array_equal(ga, gb), "chunk %d step %d env %d" % (chunk, step, i)
        for s in ref + got:
            emu.emu_destroy(s)


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="no nvcc")
def test_persist_kernel_cross_compiles_for_sm90a(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(ROOT, "loco_mujoco_b200", "csrc", "locosim.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-prec-div=false",
                        "-prec-sqrt=false", "-ftz=true", "-Xptxas", "-v", "-cubin", "-o", str(tmp_path / "locosim.cubin"), src],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    split, persist = _ptxas_report(r.stderr, "substep_kernel"), _ptxas_report(r.stderr, "persist_kernel")
    assert set(persist) == set(split), (split, persist)
    # the path it replaces by default: one resident block of 15 warps per SM needs <= 128 registers, and the stack (spills
    # of the __noinline__ phases) must not grow
    ell = "11CfgEllEuler"
    assert persist[ell][0] <= 128 and persist[ell][1] <= split[ell][1], (split[ell], persist[ell])


# ---------------------------------------------------------------------------------------------------------------------
# GPU tier
# ---------------------------------------------------------------------------------------------------------------------
def _rollout(knobs, task, n, steps, kw, monkeypatch):
    import torch
    for k, v in knobs.items():
        monkeypatch.setenv(k, str(v))
    env = make_env(task, num_envs=n, seed=5, **kw)
    eng = env._get_engine()
    nu = env.info.action_space.shape[0]
    out = [env.reset().clone()]
    g = torch.Generator(device="cpu").manual_seed(7)
    n_done = 0
    for _ in range(steps):
        act = (torch.rand((n, nu), generator=g) * 2 - 1).cuda()
        obs, rew, done, info = env.step(act)
        out += [obs.clone(), rew.clone(), done.clone(), info["next_obs"].clone()]
        n_done += int(done.sum())
    q, v, w = eng.get_state()
    cnt = eng.counters()
    out += [q.clone(), v.clone(), w.clone(), cnt[:, 0:5].clone()]
    torch.cuda.synchronize()
    for k in knobs:
        monkeypatch.delenv(k)
    return out, n_done, eng.kernels_per_step, cnt


CASES = [("UnitreeA1.simple", 4096, {}, [{}]),                                  # the default path of the headline workload
         ("UnitreeA1.simple", 2000, {"warps_per_block": 15},                    # partial last group: ghost warps
          [{"LOCOSIM_PERSIST": 1, "LOCOSIM_RESORT": s} for s in (1, 2, 3)]),
         ("UnitreeA1.simple", 2000, {}, [{"LOCOSIM_PERSIST_GRID": 3}]),        # fewer blocks than SMs
         ("UnitreeA1.simple", 4096, {}, [{"LOCOSIM_PERSIST_POOL": 0}, {"LOCOSIM_PERSIST_POOL": 8}]),
         ("UnitreeA1.simple", 2000, {"use_foot_forces": True}, [{"LOCOSIM_PERSIST": 1, "LOCOSIM_RESORT": 2}]),
         ("UnitreeA1.simple", 2000, {"reward_type": "tracking"}, [{"LOCOSIM_PERSIST": 1, "LOCOSIM_RESORT": 2}]),
         ("Talos.walk", 2000, {"domain_randomization_config": "domain_randomization_talos.yaml"},
          [{"LOCOSIM_PERSIST": 1, "LOCOSIM_RESORT": 2}])]


@pytest.mark.gpu
@pytest.mark.parametrize("task,n,kw,variants", CASES,
                         ids=["A1-4096-default", "A1-2000-chunks", "A1-grid3", "A1-pool", "A1-foot-forces", "A1-tracking",
                              "Talos-DR"])
def test_persistent_kernel_is_bitwise_identical(bundled_only, monkeypatch, task, n, kw, variants):
    import torch
    ref, n_done, kps, _ = _rollout({"LOCOSIM_RESORT": 100, "LOCOSIM_PERSIST": 0}, task, n, 50, kw, monkeypatch)
    assert n_done > 0, "the rollout should reach the auto-reset path"
    assert kps == 2, "the reference is the fused kernel with its regrouping kernel"
    for knobs in variants:
        got, _, kps, cnt = _rollout(knobs, task, n, 50, kw, monkeypatch)
        assert kps == 1, (knobs, "one persistent launch per step")
        assert bool((cnt[:, 0] == 50).all()), (knobs, "every env stepped once per control step")
        for i, (a, b) in enumerate(zip(ref, got)):
            assert torch.equal(a, b), "%s differs from the fused kernel in output %d" % (knobs, i)


@pytest.mark.gpu
def test_persistent_kernel_replays_in_a_cuda_graph(bundled_only, monkeypatch):
    """Three steps captured once and replayed twice (the queue's step parity is kept on the device) equal eager steps."""
    import torch
    monkeypatch.setenv("LOCOSIM_PERSIST", "1")
    n = 2000
    envs = [make_env("UnitreeA1.simple", num_envs=n, seed=3) for _ in range(2)]
    engs = [e._get_engine() for e in envs]
    assert all(e.kernels_per_step == 1 for e in engs)
    g = torch.Generator(device="cpu").manual_seed(11)
    acts = [(torch.rand((n, 12), generator=g) * 2 - 1).cuda() for _ in range(3)]
    for e in engs:
        e.reset()
        for _ in range(5):                       # one step outside the capture on each engine first
            e.step(acts[0])
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for a in acts:
            engs[1].step(a)
    for rep in range(2):
        for a in acts:
            o0, r0, d0, n0 = engs[0].step(a)
        graph.replay()
        torch.cuda.synchronize()
        o1, r1, d1, n1 = engs[1].obs, engs[1].reward, engs[1].done, engs[1].next_obs
        for a, b in zip((o0, r0, d0, n0) + engs[0].get_state(), (o1, r1, d1, n1) + engs[1].get_state()):
            assert torch.equal(a, b), "replay %d" % rep
        assert torch.equal(engs[0].counters()[:, :5], engs[1].counters()[:, :5])
