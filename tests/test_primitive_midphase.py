"""The lean primitive mid-phase of UnitreeA1's configuration (locosim_core.cuh collision(), CfgEllEuler::PRIMLEAN).

With PRIMLEAN the primitive pairs are filtered in one lean pass and the narrow phase runs once per 32 compacted hits,
instead of after every round of 32 filtered pairs; LOCOSIM_DEBUG bit 64 runs the rounds instead. The contact list must be
the same bit for bit either way. CPU tier: the sm_90a cross-compile with -Xptxas -v, with the flag and without it
(-DLOCOSIM_PRIMLEAN=0): A1's kernels keep their registers, stack and spills, and the other configurations do not change.
GPU tier: an elliptic-cone capacity model (more than 32 hits, so two narrow sets, and the 16-contact cap inside the first
set) against the serial build, and UnitreeA1 rollouts that must be byte-identical with the lean pass on and off."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT

ROUNDS = 64                # LOCOSIM_DEBUG bit: primitive pairs in rounds of 32 (the path without PRIMLEAN)
ELL = "11CfgEllEuler"
OTHERS = ("11CfgPyrEuler", "9CfgPyrRK4", "13CfgPyrEuler29")


# ---------------------------------------------------------------------------------------------------------------------
# CPU tier
# ---------------------------------------------------------------------------------------------------------------------
def _ptxas(stderr):
    """{function: [(registers or None, stack, spill stores, spill loads), ...]} from ptxas -v, entries and __noinline__
    functions alike (a __noinline__ function is reported once per kernel that calls it)."""
    out, cur = {}, None
    for line in stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'|Function properties for (\S+)", line)
        if m:
            cur = m.group(1) or m.group(2)
            out.setdefault(cur, [])
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur].append([None] + [int(x) for x in m.groups()])
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur and out[cur]:
            out[cur][-1][0] = int(m.group(1))
    return {k: [tuple(x) for x in v] for k, v in out.items()}


@pytest.fixture(scope="module")
def ptxas_reports(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    tmp = tmp_path_factory.mktemp("primlean")
    src = os.path.join(ROOT, "loco_mujoco_b200", "csrc", "locosim.cu")
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-prec-div=false", "-prec-sqrt=false",
             "-ftz=true", "-Xptxas", "-v", "-cubin"]
    procs = {on: subprocess.Popen([nvcc] + flags + ["-DLOCOSIM_PRIMLEAN=%d" % on, "-o", str(tmp / ("p%d.cubin" % on)), src],
                                  stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for on in (0, 1)}
    reps = {}
    for on, p in procs.items():
        _, err = p.communicate()
        assert p.returncode == 0, err[-4000:]
        reps[on] = _ptxas(err)
    return reps


def _kernel(rep, kind, cfg):
    ks = [k for k in rep if k.startswith("_Z%d%sI%s" % (len(kind), kind, cfg))]
    assert len(ks) == 1, (kind, cfg, ks)
    (entry,) = rep[ks[0]]
    return entry


def test_a1_kernels_keep_registers_stack_and_spills(ptxas_reports):
    """Every A1 kernel (fused, sub-step, persistent) fits 128 registers, the persistent kernel's stack is no larger than
    the sub-step kernel's, and every A1 kernel and __noinline__ stage reports no more registers, stack or spills with the
    lean pass than without it."""
    on, off = ptxas_reports[1], ptxas_reports[0]
    for kind in ("step_kernel", "substep_kernel", "persist_kernel"):
        regs, stack, st, ld = _kernel(on, kind, ELL)
        assert regs <= 128, (kind, regs)
    p, s = _kernel(on, "persist_kernel", ELL), _kernel(on, "substep_kernel", ELL)
    assert p[1] <= s[1], (p, s)
    a1 = [k for k in on if ELL in k]
    assert any("collision" in k for k in a1)
    for k in a1:
        assert len(on[k]) == len(off.get(k, [])), k
        for x, y in zip(on[k], off[k]):
            assert (x[0] or 0) <= (y[0] or 0) and x[1] <= y[1] and x[2] <= y[2] and x[3] <= y[3], (k, x, y)


def test_other_configurations_do_not_change(ptxas_reports):
    """The flag is A1's alone: every kernel and stage of the other configurations reports the same registers, stack and
    spills whether A1's configuration has it or not."""
    on, off = ptxas_reports[1], ptxas_reports[0]
    others = [k for k in set(on) | set(off) if ELL not in k and any(c in k for c in OTHERS)]
    assert len(others) > 20
    for k in others:
        assert on.get(k) == off.get(k), (k, on.get(k), off.get(k))


# ---------------------------------------------------------------------------------------------------------------------
# GPU tier
# ---------------------------------------------------------------------------------------------------------------------
CAPACITY_ELL_XML = """
<mujoco model="capacity_elliptic">
  <option timestep="0.002" integrator="Euler" cone="elliptic"/>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 1" condim="3"/>
    <body name="base" pos="0 0 0.05">
      <joint name="bz" type="slide" axis="0 0 1"/>
      {base}
      <body name="carriage" pos="0 0 0">
        <joint name="cx" type="slide" axis="1 0 0"/>
        <geom name="c_mass" type="sphere" size="0.01" mass="0.1" contype="0" conaffinity="0"/>
        <body name="probe" pos="0 0 0.3">
          <joint name="pz" type="slide" axis="0 0 1"/>
          {probe}
        </body>
      </body>
    </body>
  </worldbody>
  <actuator>
    <motor name="m_cx" joint="cx" gear="1"/>
  </actuator>
</mujoco>
"""
N_BASE, N_PROBE = 30, 6


def capacity_model_elliptic():
    """30 condim-6 spheres on the base and 6 on the probe (grandchild of the base), all sunk 2-4 cm into the floor, each
    probe sphere 3 cm beside a base sphere: 36 floor pairs and some sphere-sphere pairs pass the filter, more than 32
    hits (two narrow sets); the floor pairs alone give one contact each, so the 16-contact cap falls inside the first set.
    The elliptic cone puts the model on UnitreeA1's configuration (CfgEllEuler)."""
    import tempfile
    from loco_mujoco_b200 import mjcf, modelpack
    pos = [(0.12 * (k % 6) - 0.30, 0.12 * (k // 6) - 0.24) for k in range(N_BASE)]
    base = "".join('<geom type="sphere" size="0.05" pos="%.3f %.3f -0.03" mass="0.2" condim="6"/>' % p for p in pos)
    probe = "".join('<geom type="sphere" size="0.05" pos="%.3f %.3f -0.33" mass="0.2" condim="6"/>'
                    % (pos[5 * k][0] + 0.03, pos[5 * k][1]) for k in range(N_PROBE))
    with tempfile.NamedTemporaryFile("w", suffix=".xml", delete=False) as f:
        f.write(CAPACITY_ELL_XML.format(base=base, probe=probe))
        path = f.name
    try:
        m = mjcf.compile_model(mjcf.XmlHandle(path), fuse_static=False)
    finally:
        os.unlink(path)
    return m, modelpack.pack(m)


def _contacts(r, i):
    n = int(r["ncon"][i])
    return [(int(r["con_g1"][i, k]), int(r["con_g2"][i, k]), int(r["con_dim"][i, k])) for k in range(n)]


@pytest.mark.gpu
def test_capacity_edges_elliptic_match_serial_build():
    """More than 32 primitive hits in one evaluation (two narrow sets) and the 16-contact cap inside the first set: the
    CUDA build drops the same contacts as the serial build (ncon_raw, ncon, contact list, r_ti), with the lean pass and
    with the rounds (LOCOSIM_DEBUG bit 64); the two CUDA runs agree bit for bit on the contacts."""
    import stage_probe as sp
    from loco_mujoco_b200.task import TaskSpec, OBS_QPOS, OBS_QVEL, REWARD_NONE
    m, mb = capacity_model_elliptic()
    S = sp.capacity_states(m)
    # every sphere's centre is below its radius: each floor pair passes the filter (36 > 32 hits)
    z_base = 0.05 + S["qpos"][:, 0] - 0.03
    z_probe = 0.05 + S["qpos"][:, 0] + 0.3 + S["qpos"][:, 2] - 0.33
    assert np.all(z_base < 0.05) and np.all(z_probe < 0.05) and N_BASE + N_PROBE > 32
    nv = m.nv
    spec = TaskSpec([OBS_QPOS] * nv + [OBS_QVEL] * nv, list(range(nv)) * 2, [], REWARD_NONE, [], [], np.zeros(m.nu), np.ones(m.nu),
                    5, np.zeros((1, 1, 2 * nv)), 0, [nv, nv], use_absorbing=False)
    lib = sp._bind(ctypes.CDLL(sp.build_cuda()))
    e, cfg = sp.emu_record(sp.build_emu(), mb, S)
    assert cfg == 0, "the elliptic model runs on CfgEllEuler"
    recs = {}
    for dbg in (0, ROUNDS):
        cp = sp.CudaProbe(lib, mb, spec.pack(), len(S["qpos"]), env_vars={"LOCOSIM_DEBUG": dbg})
        assert cp.cfg == cfg
        recs[dbg] = sp.decode(lib, cp.run(S))
        cp.close()
    for g in (e, recs[0], recs[ROUNDS]):
        assert np.all(g["ncon_raw"] == 16)
    for g in (recs[0], recs[ROUNDS]):
        for f in ("ncon_raw", "ncon", "nunit", "nrow", "nefc"):
            assert np.array_equal(e[f], g[f]), f
        for i in range(len(S["qpos"])):
            assert _contacts(e, i) == _contacts(g, i), i
            nefc = int(g["nefc"][i])
            assert np.array_equal(e["r_ti"][i, :nefc], g["r_ti"][i, :nefc]), i
    for f in ("con_g1", "con_g2", "con_dist", "con_pos", "con_frame", "con_incl"):
        assert np.array_equal(recs[0][f], recs[ROUNDS][f]), f
    print("elliptic capacity model: ncon_raw 16, ncon %s, nrow %s" % (sorted(set(e["ncon"])), sorted(set(e["nrow"]))))


_GPU_SCRIPT = r"""
import os, sys, torch
sys.path.insert(0, sys.argv[1])
os.environ["LOCO_MUJOCO_B200_FORCE_BUNDLED"] = "1"
from loco_mujoco_b200 import LocoEnv
n = int(sys.argv[3])
env = LocoEnv.make("UnitreeA1.simple", num_envs=n, seed=5)
eng = env._get_engine()
cw = env.contact_wrench                                         # registers the contact outputs
g = torch.Generator(device=eng.device).manual_seed(11)
acts = torch.rand((50, eng.n_envs, eng.action_dim), device=eng.device, generator=g) * 2 - 1
eng.reset()
outs, resets = [], 0
for k in range(50):
    obs, rew, done, nxt = eng.step(acts[k])
    outs += [obs.clone(), rew.clone(), done.clone(), nxt.clone(), cw.clone()]
    resets += int(done.sum())
    if k % 10 == 9:
        outs += [x.clone() for x in eng.get_state()]           # qpos, qvel, warm start
torch.cuda.synchronize()
torch.save({"outs": [o.cpu() for o in outs], "info": str(eng.launch_info()), "resets": resets}, sys.argv[2])
"""


@pytest.mark.gpu
@pytest.mark.parametrize("n,knobs", [(4096, {}), (2000, {}), (4096, {"LOCOSIM_PERSIST": 0, "LOCOSIM_RESORT": 10})],
                         ids=["4096-persistent", "2000-ghost-warps", "4096-fused"])
def test_gpu_steps_are_unchanged_by_the_lean_midphase(tmp_path, n, knobs):
    """50 auto-resetting steps of UnitreeA1: outputs, qpos, qvel, warm start and the registered contact_wrench are
    byte-identical with the lean primitive pass and with the rounds (LOCOSIM_DEBUG bit 64)."""
    import torch
    script = tmp_path / "run.py"
    script.write_text(_GPU_SCRIPT)
    res = {}
    for dbg in (ROUNDS, 0):
        out = tmp_path / ("run%d.pt" % dbg)
        env = dict(os.environ, LOCOSIM_DEBUG=str(dbg), **{k: str(v) for k, v in knobs.items()})
        subprocess.check_call([sys.executable, str(script), ROOT, str(out), str(n)], env=env)
        res[dbg] = torch.load(out)
    a, b = res[0], res[ROUNDS]
    print(a["info"])
    assert len(a["outs"]) == len(b["outs"]) == 50 * 5 + 5 * 3
    assert a["resets"] > 0, "the rollout should reach the auto-reset path"
    assert float(a["outs"][4].abs().max()) > 0, "contacts reach the registered outputs"
    for k, (x, y) in enumerate(zip(a["outs"], b["outs"])):
        assert torch.equal(x, y), k
