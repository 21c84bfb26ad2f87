"""
ctypes binding of the CUDA engine's C-ABI (include/locosim.h -> loco_mujoco_b200/liblocosim_cuda.so).

There is NO CPU fallback: if the shared library is missing or no CUDA device is visible, constructing an engine
raises. (The fp64 CPU oracle under oracle/ is test infrastructure and is never imported from here.)
"""
import ctypes
import math
import os

import numpy as np

_LIB = None
_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "liblocosim_cuda.so")


class EngineUnavailable(RuntimeError):
    pass


def load_library():
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(_LIB_PATH):
        raise EngineUnavailable("CUDA engine library not built: %s (run `python -c 'import __graft_entry__ as g; "
                                "g.build()'`)" % _LIB_PATH)
    lib = ctypes.CDLL(_LIB_PATH)
    vp, ip = ctypes.c_void_p, ctypes.c_int
    lib.locosim_create.restype = ip
    lib.locosim_create.argtypes = [vp, ip, vp, ip, vp, ip, vp, ip, ip, ip, ctypes.c_uint64, ctypes.c_int64,
                                   ctypes.POINTER(vp)]
    lib.locosim_destroy.restype = None
    lib.locosim_destroy.argtypes = [vp]
    lib.locosim_last_error.restype = ctypes.c_char_p
    lib.locosim_last_error.argtypes = [vp]
    for name in ("locosim_num_envs", "locosim_obs_dim", "locosim_action_dim", "locosim_nq"):
        getattr(lib, name).restype = ip
        getattr(lib, name).argtypes = [vp]
    lib.locosim_set_solver.restype = ip
    lib.locosim_set_solver.argtypes = [vp, ctypes.c_float, ctypes.c_float, ip, ip]
    lib.locosim_reset.restype = ip
    lib.locosim_reset.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.locosim_reset_rows.restype = ip
    lib.locosim_reset_rows.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.locosim_step.restype = ip
    lib.locosim_step.argtypes = [vp, vp, vp, vp, vp, vp, ip, vp]
    lib.locosim_get_state.restype = ip
    lib.locosim_get_state.argtypes = [vp, vp, vp, vp, vp]
    lib.locosim_set_state.restype = ip
    lib.locosim_set_state.argtypes = [vp, vp, vp, vp, vp]
    lib.locosim_set_reset_rotation.restype = ip
    lib.locosim_set_reset_rotation.argtypes = [vp, vp]
    lib.locosim_get_cursor.restype = ip
    lib.locosim_get_cursor.argtypes = [vp, vp, vp]
    lib.locosim_dataset_rows.restype = ip
    lib.locosim_dataset_rows.argtypes = [vp]
    lib.locosim_create_dataset.restype = ip
    lib.locosim_create_dataset.argtypes = [vp, vp, vp, vp, vp]
    lib.locosim_set_goal.restype = ip
    lib.locosim_set_goal.argtypes = [vp, vp, vp]
    lib.locosim_get_counters.restype = ip
    lib.locosim_get_counters.argtypes = [vp, vp, vp]
    lib.locosim_param_pool_row_len.restype = ip
    lib.locosim_param_pool_row_len.argtypes = [vp]
    lib.locosim_set_param_pool.restype = ip
    lib.locosim_set_param_pool.argtypes = [vp, vp, ip, ip]
    lib.locosim_get_param_rows.restype = ip
    lib.locosim_get_param_rows.argtypes = [vp, vp, vp]
    lib.locosim_kernels_per_step.restype = ip
    lib.locosim_kernels_per_step.argtypes = [vp]
    lib.locosim_measure_fp32_peak.restype = ip
    lib.locosim_measure_fp32_peak.argtypes = [ip, ctypes.POINTER(ctypes.c_double)]
    lib.locosim_launch_info.restype = ip
    lib.locosim_launch_info.argtypes = [vp, ctypes.POINTER(ip), ctypes.POINTER(ip), ctypes.POINTER(ip)]
    lib.locosim_set_timeline.restype = ip
    lib.locosim_set_timeline.argtypes = [vp, vp, ip]
    lib.locosim_set_time_limit.restype = ip
    lib.locosim_set_time_limit.argtypes = [vp, ip, ip]
    lib.locosim_get_episode_stats.restype = ip
    lib.locosim_get_episode_stats.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.locosim_nbody.restype = ip
    lib.locosim_nbody.argtypes = [vp]
    lib.locosim_set_applied_forces.restype = ip
    lib.locosim_set_applied_forces.argtypes = [vp, vp, vp]
    lib.locosim_set_terrain_origin.restype = ip
    lib.locosim_set_terrain_origin.argtypes = [vp, vp]
    lib.locosim_set_body_outputs.restype = ip
    lib.locosim_set_body_outputs.argtypes = [vp, vp, vp]
    lib.locosim_set_contact_outputs.restype = ip
    lib.locosim_set_contact_outputs.argtypes = [vp, vp]
    lib.locosim_set_dof_outputs.restype = ip
    lib.locosim_set_dof_outputs.argtypes = [vp, vp]
    lib.locosim_set_reference_outputs.restype = ip
    lib.locosim_set_reference_outputs.argtypes = [vp, vp, vp]
    lib.locosim_create_dataset_bodies.restype = ip
    lib.locosim_create_dataset_bodies.argtypes = [vp, vp, vp, vp]
    lib.locosim_inverse.restype = ip
    lib.locosim_inverse.argtypes = [vp, vp, vp, vp]
    lib.locosim_create_dataset_inverse.restype = ip
    lib.locosim_create_dataset_inverse.argtypes = [vp, vp, vp]
    lib.locosim_dynamics_terms.restype = ip
    lib.locosim_dynamics_terms.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    lib.locosim_forward.restype = ip
    lib.locosim_forward.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.locosim_state_words.restype = ip
    lib.locosim_state_words.argtypes = [vp]
    lib.locosim_max_contacts.restype = ip
    lib.locosim_max_contacts.argtypes = [vp]
    lib.locosim_set_contact_list_outputs.restype = ip
    lib.locosim_set_contact_list_outputs.argtypes = [vp, vp, vp, vp]
    lib.locosim_save_state.restype = ip
    lib.locosim_save_state.argtypes = [vp, vp, vp, vp]
    lib.locosim_load_state.restype = ip
    lib.locosim_load_state.argtypes = [vp, vp, ip, vp, vp, vp]
    lib.locosim_ray.restype = ip
    lib.locosim_ray.argtypes = [vp, vp, vp, ip, ip, ip, ip, ip, vp, vp, vp, vp]
    _LIB = lib
    return lib


EXPORTED_SYMBOLS = ["locosim_create", "locosim_destroy", "locosim_last_error", "locosim_num_envs", "locosim_obs_dim",
                    "locosim_action_dim", "locosim_nq", "locosim_set_solver", "locosim_reset", "locosim_step",
                    "locosim_get_state", "locosim_set_state", "locosim_get_counters", "locosim_launch_info",
                    "locosim_param_pool_row_len", "locosim_set_param_pool", "locosim_get_param_rows",
                    "locosim_kernels_per_step", "locosim_reset_rows", "locosim_set_goal", "locosim_measure_fp32_peak",
                    "locosim_set_reset_rotation", "locosim_get_cursor", "locosim_dataset_rows", "locosim_create_dataset",
                    "locosim_debug_counters", "locosim_set_timeline", "locosim_set_time_limit",
                    "locosim_get_episode_stats", "locosim_nbody", "locosim_set_applied_forces",
                    "locosim_set_body_outputs", "locosim_set_contact_outputs", "locosim_set_dof_outputs",
                    "locosim_set_reference_outputs", "locosim_create_dataset_bodies", "locosim_inverse",
                    "locosim_create_dataset_inverse", "locosim_dynamics_terms", "locosim_forward", "locosim_state_words",
                    "locosim_save_state", "locosim_load_state", "locosim_max_contacts",
                    "locosim_set_contact_list_outputs", "locosim_ray", "locosim_set_terrain_origin"]

# values per body row of the body outputs (include/locosim.h LS_BODY_DIM): xpos (3), xquat w x y z (4), angular velocity (3),
# linear velocity of the body-frame origin (3), world frame
BODY_DIM = 13
# values per body row of the contact outputs (include/locosim.h LS_CONTACT_DIM): force (3), torque about xpos (3), world frame
CONTACT_DIM = 6
# values per dof row of the dof outputs (include/locosim.h LS_DOF_DIM): qfrc_actuator, qfrc_constraint, qacc
DOF_DIM = 3
# values per env of the dynamics terms' centre of mass (include/locosim.h LS_COM_DIM): x, y, z, total mass
COM_DIM = 4
# values per body row of the forward dynamics' body accelerations (include/locosim.h LS_BODY_ACC_DIM): angular acceleration
# (3), linear acceleration of the body-frame origin minus gravity (3), world frame
BODY_ACC_DIM = 6
# values per contact row of the contact list (include/locosim.h LS_CONLIST_DIM / LS_CONLIST_ID_DIM) and their columns
# (LS_CONLIST_*): dist (1), pos (3), frame rows n, t1, t2 (9), contact-frame force (6); geom1, geom2, body1, body2, dim
CONLIST_DIM = 19
CONLIST_COLUMNS = dict(dist=(0, 1), pos=(1, 3), frame=(4, 9), force=(13, 6))
CONLIST_ID_DIM = 5
CONLIST_ID_COLUMNS = dict(geom=(0, 2), body=(2, 2), dim=(4, 1))
# ray query frames and flags (include/locosim.h LS_RAY_*): where pnt / vec are given, and which geoms a ray can hit
RAY_WORLD, RAY_BODY, RAY_HEADING, RAY_TRACK = 0, 1, 2, 3
RAY_STATIC, RAY_DYNAMIC, RAY_PER_ENV = 1, 2, 4
# rays per env of one locosim_ray launch: 65535 blocks of 128 (include/locosim.h)
RAY_MAX = 65535 * 128



def state_layout(nq, obs_dim):
    """{field: (offset, length)} of a saved-state row (include/locosim.h LS_STATE_*), int32 words; "words" is the row length
    W. Fields stored as fp32 (angle, ep[1], ep[3], goal, qpos, qvel, qacc_warmstart, obs) are read with `.view(float32)`."""
    return dict(tag=(0, 2), episode=(2, 1), dr_row=(3, 1), cursor=(4, 1), angle=(5, 1), ep=(8, 4), goal=(12, 4),
                qpos=(16, nq), qvel=(16 + nq, nq), qacc_warmstart=(16 + 2 * nq, nq), obs=(16 + 3 * nq, obs_dim),
                words=(0, (16 + 3 * nq + obs_dim + 3) // 4 * 4))


# bits of the done byte of a step (include/locosim.h)
DONE_ABSORBING, DONE_TRUNCATED = 1, 2


def split_done(done):
    """done bytes of a step -> (absorbing, truncated) bool masks (torch or numpy uint8 in, the same kind out)."""
    return (done & DONE_ABSORBING) != 0, (done & DONE_TRUNCATED) != 0


def measure_fp32_peak(device=0):
    """Measured non-tensor FP32 FMA peak of the device in TFLOP/s (include/locosim.h)."""
    v = ctypes.c_double(0)
    if load_library().locosim_measure_fp32_peak(int(device), ctypes.byref(v)) != 0:
        raise RuntimeError("locosim_measure_fp32_peak failed")
    return v.value


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class CudaEngine:
    """n_envs independent worlds of one compiled model on one GPU; all I/O are torch.cuda tensors."""

    def __init__(self, model_blobs, task_blobs, n_envs, device=0, seed=0, env_id_offset=0, warps_per_block=None):
        import torch
        if not torch.cuda.is_available():
            raise EngineUnavailable("no CUDA device visible: the locosim engine has no CPU path")
        self.torch = torch
        self.lib = load_library()
        mi, mr = model_blobs
        ti, tr = task_blobs
        mi = np.ascontiguousarray(mi, dtype=np.int32)
        mr = np.ascontiguousarray(mr, dtype=np.float64)
        ti = np.ascontiguousarray(ti, dtype=np.int32)
        tr = np.ascontiguousarray(tr, dtype=np.float64)
        h = ctypes.c_void_p()
        # launch geometry: envs (= warps) per block; None = the engine's own choice (the largest block that keeps the most
        # envs resident per SM). Smaller blocks let several engines share an SM (MixedBatch). Scheduling only.
        prev = os.environ.get("LOCOSIM_WPB")
        if warps_per_block is not None:
            os.environ["LOCOSIM_WPB"] = str(int(warps_per_block))
        try:
            rc = self._create(mi, mr, ti, tr, n_envs, device, seed, env_id_offset, h)
        finally:
            if warps_per_block is not None:
                if prev is None:
                    os.environ.pop("LOCOSIM_WPB", None)
                else:
                    os.environ["LOCOSIM_WPB"] = prev
        if rc != 0:
            raise RuntimeError("locosim_create failed: %s" % self.lib.locosim_last_error(None).decode())
        self._finish_init(h, n_envs, device)

    def _create(self, mi, mr, ti, tr, n_envs, device, seed, env_id_offset, h):
        return self.lib.locosim_create(mi.ctypes.data, len(mi), mr.ctypes.data, len(mr), ti.ctypes.data, len(ti),
                                       tr.ctypes.data, len(tr), int(n_envs), int(device), int(seed), int(env_id_offset),
                                       ctypes.byref(h))

    def _finish_init(self, h, n_envs, device):
        torch = self.torch
        self.h = h
        self.device = torch.device("cuda", device)
        self.n_envs = int(n_envs)
        self.obs_dim = self.lib.locosim_obs_dim(h)
        self.action_dim = self.lib.locosim_action_dim(h)
        self.nq = self.lib.locosim_nq(h)
        self.nbody = self.lib.locosim_nbody(h)
        self._applied = (None, None)      # the registered applied-force tensors (kept alive while registered)
        self._body_out = (None, None)     # the registered body-output tensors (likewise)
        self._contact_out = None          # the registered contact-output tensor (likewise)
        self._dof_out = None              # the registered dof-output tensor (likewise)
        self._conlist_out = (None, None, None)   # the registered contact-list tensors (likewise)
        self._ref_out = (None, None)      # the registered reference-output tensors (likewise)
        # obs / reward / done of a step live in ONE device allocation (three views), so that a consumer on the host can
        # fetch the whole step result with a single D2H copy of `packed_out`
        N, D = int(n_envs), self.obs_dim
        self.packed_out = torch.zeros((N * (4 * D + 5),), dtype=torch.uint8, device=self.device)
        self.obs, self.reward, self.done = self.views_of(self.packed_out)
        self.next_obs = torch.zeros((n_envs, self.obs_dim), dtype=torch.float32, device=self.device)
        self.launches = 0
        self.kernels_per_step = self.lib.locosim_kernels_per_step(h)
        self.state_words = self.lib.locosim_state_words(h)
        self.max_contacts = self.lib.locosim_max_contacts(h)

    def views_of(self, packed):
        """(obs [N, D] f32, reward [N] f32, done [N] u8) views of a buffer laid out like `packed_out`."""
        N, D, t = self.n_envs, self.obs_dim, self.torch
        return (packed[:4 * N * D].view(t.float32).view(N, D), packed[4 * N * D:4 * N * D + 4 * N].view(t.float32),
                packed[4 * N * D + 4 * N:])

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError("locosim: %s" % self.lib.locosim_last_error(self.h).decode())

    def _check_tensor(self, x, name, shape, dtype="float32"):
        """Refuse `x` (ValueError naming it) unless it is a contiguous tensor of `dtype` (float32 or int32) on this
        engine's device of exactly `shape`: the engine reads or writes every env's whole rows through its pointer. Anything
        without a tensor's dtype / is_contiguous / device / shape (None, a numpy array) is refused as well."""
        t = self.torch
        if not all(hasattr(x, a) for a in ("dtype", "is_contiguous", "device", "shape")) or x.dtype != getattr(t, dtype) \
                or not x.is_contiguous() or x.device != self.device:
            raise ValueError("%s must be a contiguous %s tensor on %s" % (name, dtype, self.device))
        if tuple(x.shape) != shape:
            raise ValueError("%s shape %s != %s" % (name, tuple(x.shape), shape))

    @staticmethod
    def _check_disjoint(spans):
        """Refuse (ValueError naming both) any two of `spans` (name, tensor, shape) whose float32 or int32 buffers overlap; a
        None tensor is skipped. Byte sizes come from the checked shapes."""
        seen = []
        for name, x, shape in spans:
            if x is None:
                continue
            a, size = x.data_ptr(), 4 * math.prod(shape)
            for other, b, bsize in seen:
                if size and bsize and a < b + bsize and b < a + size:
                    raise ValueError("%s and %s must not overlap" % (other, name))
            seen.append((name, a, size))

    def _stream(self):
        return ctypes.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def close(self):
        if getattr(self, "h", None):
            self.lib.locosim_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_solver(self, tolerance=1e-5, ls_tolerance=0.1, max_iter=20, ls_iter=16):
        self._check(self.lib.locosim_set_solver(self.h, tolerance, ls_tolerance, max_iter, ls_iter))

    def reset(self, mask=None, traj_no=None, step_no=None, out=None, pool_row=None, rot_angle=None):
        """rot_angle: float32 cuda [n_envs], rotation angles of this reset (setup_random_rot with host-drawn angles)."""
        out = self.next_obs if out is None else out
        if rot_angle is not None:
            self._check(self.lib.locosim_set_reset_rotation(self.h, _ptr(rot_angle)))
        self._check(self.lib.locosim_reset_rows(self.h, _ptr(mask), _ptr(traj_no), _ptr(step_no), _ptr(pool_row), _ptr(out),
                                                self._stream()))
        self.launches += 1 if self._body_out[1] is None and self._ref_out == (None, None) else 2
        return out

    @property
    def packed_bytes(self):
        """Bytes of one step's (obs f32 [N, D] | reward f32 [N] | done u8 [N]) record."""
        return self.n_envs * (4 * self.obs_dim + 5)

    def step(self, action, auto_reset=True, want_next_obs=True, packed=None):
        """action: float32 cuda [n_envs, action_dim] (contiguous). Returns (obs, reward, done, next_obs) views; `done` is the
        engine's byte (bit 0 absorbing, bit 1 truncated by `set_time_limit`: `split_done`).
        packed: optional uint8 cuda buffer of `packed_bytes` (16-byte aligned, e.g. one time slot of a rollout buffer)
        the kernel writes this step's obs / reward / done into instead of the engine's own `packed_out`."""
        self._check_tensor(action, "action", (self.n_envs, self.action_dim))
        if packed is None:
            obs, reward, done = self.obs, self.reward, self.done
        else:
            if packed.dtype != self.torch.uint8 or packed.numel() != self.packed_bytes or not packed.is_contiguous() \
                    or packed.data_ptr() % 4:
                raise ValueError("packed must be a contiguous, 4-byte aligned uint8 buffer of %d bytes" % self.packed_bytes)
            obs, reward, done = self.views_of(packed)
        self._check(self.lib.locosim_step(self.h, _ptr(action), _ptr(obs), _ptr(reward), _ptr(done),
                                          _ptr(self.next_obs) if want_next_obs else None, int(bool(auto_reset)),
                                          self._stream()))
        self.launches += self.kernels_per_step
        return obs, reward, done, self.next_obs

    def get_state(self):
        t = self.torch
        q = t.empty((self.n_envs, self.nq), dtype=t.float32, device=self.device)
        v = t.empty_like(q)
        w = t.empty_like(q)
        self._check(self.lib.locosim_get_state(self.h, _ptr(q), _ptr(v), _ptr(w), self._stream()))
        return q, v, w

    def set_state(self, qpos, qvel, qacc_warmstart=None):
        for x, name in ((qpos, "qpos"), (qvel, "qvel"), (qacc_warmstart, "qacc_warmstart")):
            if x is not None:
                self._check_tensor(x, name, (self.n_envs, self.nq))
        self._check(self.lib.locosim_set_state(self.h, _ptr(qpos), _ptr(qvel), _ptr(qacc_warmstart), self._stream()))

    def set_time_limit(self, max_episode_steps=0, end_of_trajectory=False):
        """Time limit of include/locosim.h: truncate an episode at `max_episode_steps` control steps (0 = no limit) and / or
        where its trajectory cursor reaches the last mocap sample. Reported as bit 1 of `done`; takes effect from the next step."""
        self._check(self.lib.locosim_set_time_limit(self.h, int(max_episode_steps), int(bool(end_of_trajectory))))

    def set_applied_forces(self, xfrc=None, qfrc=None):
        """Register the applied forces of include/locosim.h (MuJoCo's xfrc_applied / qfrc_applied): `xfrc` float32 cuda
        [n_envs, nbody, 6] (force then torque, world frame, at each body's centre of mass; body 0 ignored), `qfrc` float32
        cuda [n_envs, nq]; either None. The engine reads the tensors in every later step, zeroes the rows of every env it
        resets, and keeps a reference to them. None, None turns the feature off. Register outside of CUDA-graph capture."""
        for x, shape, name in ((xfrc, (self.n_envs, self.nbody, 6), "xfrc"), (qfrc, (self.n_envs, self.nq), "qfrc")):
            if x is not None:
                self._check_tensor(x, name, shape)
        self._check(self.lib.locosim_set_applied_forces(self.h, _ptr(xfrc), _ptr(qfrc)))
        self._applied = (xfrc, qfrc)

    def set_terrain_origin(self, origin=None):
        """Register the terrain origin of include/locosim.h (locosim_set_terrain_origin): `origin` float32 cuda [n_envs, 2],
        the terrain point (x, y) under each env's world origin, read by every later step and query; None = all zeros. The
        engine keeps a reference to it. Only for a model with a terrain (loco_mujoco_b200.terrain). Register outside of
        CUDA-graph capture."""
        if origin is not None:
            self._check_tensor(origin, "origin", (self.n_envs, 2))
        self._check(self.lib.locosim_set_terrain_origin(self.h, _ptr(origin)))
        self._terrain_origin = origin

    def set_body_outputs(self, body=None, next_body=None):
        """Register the body outputs of include/locosim.h (MuJoCo's xpos / xquat / body velocity): `body` and `next_body`
        float32 cuda [n_envs, nbody, BODY_DIM], either None. Every step writes `body` for the state `obs` describes (zeros for
        a non-finite env) and `next_body` for the state to act on next (after the auto-reset); reset() and set_state() write
        `next_body` as well. The engine keeps a reference to them. None, None turns the feature off. Register outside of
        CUDA-graph capture, and capture a step again after turning the feature on: whether a step writes the rows is fixed
        when it is captured (a graph captured with nothing registered writes only the terminal rows of the envs it resets;
        one captured with buffers registered writes into whatever buffers are registered at each replay)."""
        for x, name in ((body, "body"), (next_body, "next_body")):
            if x is not None:
                self._check_tensor(x, name, (self.n_envs, self.nbody, BODY_DIM))
        self._check(self.lib.locosim_set_body_outputs(self.h, _ptr(body), _ptr(next_body)))
        self._body_out = (body, next_body)
        self.kernels_per_step = self.lib.locosim_kernels_per_step(self.h)     # (+1 while registered: body_kernel)

    def set_reference_outputs(self, ref=None, next_ref=None):
        """Register the reference outputs of include/locosim.h (the mocap clip's body outputs): `ref` and `next_ref` float32
        cuda [n_envs, nbody, BODY_DIM], either None. A reference row is the body-output row of the state a reset onto the
        table row at the env's cursor gives (root x / y zeroed; the rotation angle of the env's episode; its parameter-pool
        row). Every step writes `ref` for the state `obs` describes (the cursor the terminal step reached for an env that
        ended, zeros for a non-finite env) and `next_ref` for the state to act on next (after the auto-reset); reset() writes
        `next_ref` as well, set_state() does not. The engine keeps a reference to them. None, None turns the feature off.
        The CUDA-graph rules are those of set_body_outputs: register outside of capture and capture a step again after
        turning the feature on."""
        for x, name in ((ref, "ref"), (next_ref, "next_ref")):
            if x is not None:
                self._check_tensor(x, name, (self.n_envs, self.nbody, BODY_DIM))
        self._check(self.lib.locosim_set_reference_outputs(self.h, _ptr(ref), _ptr(next_ref)))
        self._ref_out = (ref, next_ref)
        self.kernels_per_step = self.lib.locosim_kernels_per_step(self.h)     # (+1 while registered: body_kernel)

    def set_contact_outputs(self, contact=None):
        """Register the contact outputs of include/locosim.h (MuJoCo's mj_contactForce summed per body): `contact` float32
        cuda [n_envs, nbody, CONTACT_DIM], or None to turn the feature off. Every step writes, per body, the world-frame force
        and torque about the body-frame origin that the body's contacts exert on it, averaged over the step's sub-steps
        (zeros for a non-finite env). reset() and set_state() leave it alone. The engine keeps a reference to it. Register
        outside of CUDA-graph capture; a step captured earlier writes the buffer registered when it is replayed."""
        if contact is not None:
            self._check_tensor(contact, "contact", (self.n_envs, self.nbody, CONTACT_DIM))
        self._check(self.lib.locosim_set_contact_outputs(self.h, _ptr(contact)))
        self._contact_out = contact

    def set_dof_outputs(self, dof=None):
        """Register the dof outputs of include/locosim.h (MuJoCo's qfrc_actuator / qfrc_constraint / qacc): `dof` float32
        cuda [n_envs, nq, DOF_DIM], or None to turn the feature off. Every step writes, per dof (the qvel layout), the actuator
        force, the constraint force and the constrained acceleration, averaged over the step's sub-steps (zeros for a
        non-finite env). reset() and set_state() leave it alone. The engine keeps a reference to it. Register outside of
        CUDA-graph capture; a step captured earlier writes the buffer registered when it is replayed."""
        if dof is not None:
            self._check_tensor(dof, "dof", (self.n_envs, self.nq, DOF_DIM))
        self._check(self.lib.locosim_set_dof_outputs(self.h, _ptr(dof)))
        self._dof_out = dof

    def set_contact_list_outputs(self, ncon=None, con=None, con_id=None):
        """Register the contact list of include/locosim.h (MuJoCo's d.contact with each contact's mj_contactForce): `ncon`
        int32 cuda [n_envs], `con` float32 cuda [n_envs, max_contacts, CONLIST_DIM] and `con_id` int32 cuda [n_envs,
        max_contacts, CONLIST_ID_DIM], all three, or none to turn the feature off. Every step writes the contacts of its
        last sub-step in list order (CONLIST_COLUMNS / CONLIST_ID_COLUMNS), zeros and ids of -1 in the rows past ncon, and
        ncon = 0 for a non-finite env. reset(), set_state() and load_state() leave them alone. The engine keeps references
        to them. Register outside of CUDA-graph capture; a step captured earlier writes the buffers registered when it is
        replayed."""
        bufs = (ncon, con, con_id)
        if any(x is None for x in bufs) and any(x is not None for x in bufs):
            raise ValueError("ncon, con and con_id must be given together (or none of them)")
        n, C = self.n_envs, self.max_contacts
        spans = (("ncon", ncon, (n,)), ("con", con, (n, C, CONLIST_DIM)), ("con_id", con_id, (n, C, CONLIST_ID_DIM)))
        if ncon is not None:
            for (name, x, shape), dtype in zip(spans, ("int32", "float32", "int32")):
                self._check_tensor(x, name, shape, dtype)
            self._check_disjoint(spans)
        self._check(self.lib.locosim_set_contact_list_outputs(self.h, _ptr(ncon), _ptr(con), _ptr(con_id)))
        self._conlist_out = bufs

    def episode_stats(self):
        """(length int32, return float32, last_length, last_return), each [n_envs]: the running episode's control steps and
        summed engine rewards, and those of the env's last finished (absorbing or truncated) episode."""
        t = self.torch
        ln, last_ln = (t.empty((self.n_envs,), dtype=t.int32, device=self.device) for _ in range(2))
        ret, last_ret = (t.empty((self.n_envs,), dtype=t.float32, device=self.device) for _ in range(2))
        self._check(self.lib.locosim_get_episode_stats(self.h, _ptr(ln), _ptr(ret), _ptr(last_ln), _ptr(last_ret), self._stream()))
        return ln, ret, last_ln, last_ret

    def cursor(self):
        t = self.torch
        c = t.empty((self.n_envs,), dtype=t.int32, device=self.device)
        self._check(self.lib.locosim_get_cursor(self.h, _ptr(c), self._stream()))
        return c

    def create_dataset(self):
        """(states, next_states, last) of the reset table in observation layout, built on the device."""
        t = self.torch
        n = self.lib.locosim_dataset_rows(self.h)
        states = t.empty((n, self.obs_dim), dtype=t.float32, device=self.device)
        nxt = t.empty_like(states)
        last = t.empty((n,), dtype=t.float32, device=self.device)
        self._check(self.lib.locosim_create_dataset(self.h, _ptr(states), _ptr(nxt), _ptr(last), self._stream()))
        self.launches += 1
        return states, nxt, last

    def create_dataset_bodies(self):
        """(body, next_body) float32 cuda [dataset rows, nbody, BODY_DIM], row-aligned with create_dataset(): the reference
        rows of each row's (traj, sample) and (traj, sample + 1), with rotation angle 0 and the compiled model's own
        parameters, built on the device."""
        t = self.torch
        n = self.lib.locosim_dataset_rows(self.h)
        body = t.empty((n, self.nbody, BODY_DIM), dtype=t.float32, device=self.device)
        nxt = t.empty_like(body)
        self._check(self.lib.locosim_create_dataset_bodies(self.h, _ptr(body), _ptr(nxt), self._stream()))
        self.launches += 1
        return body, nxt

    def inverse(self, qacc, out=None):
        """Inverse dynamics of include/locosim.h (MuJoCo 2.3.7's continuous-time mj_inverse) of every env at its stored
        state and parameter-pool row: qfrc_inverse = M qacc + bias - passive - J^T efc_force(J qacc - aref), actuator and
        applied forces not subtracted. `qacc` float32 cuda [n_envs, nq] (the qvel layout); `out` float32 cuda [n_envs, nq]
        not overlapping it, or None for a new tensor. A non-finite state or qacc gives that env a row of zeros. Changes
        nothing else in the engine; stream-ordered, no allocation when `out` is given (can be captured in a CUDA graph)."""
        t = self.torch
        shape = (self.n_envs, self.nq)
        if out is None:
            out = t.empty(shape, dtype=t.float32, device=self.device)
        self._check_tensor(qacc, "qacc", shape)
        self._check_tensor(out, "out", shape)
        self._check_disjoint((("qacc", qacc, shape), ("out", out, shape)))
        self._check(self.lib.locosim_inverse(self.h, _ptr(qacc), _ptr(out), self._stream()))
        self.launches += 1
        return out

    def create_dataset_inverse(self):
        """float32 cuda [dataset rows, nq], row-aligned with create_dataset(): row r is the inverse dynamics at the reset
        state of its (traj, sample) (rotation angle 0, the compiled model's own parameters) at the forward-difference
        acceleration qacc = (qvel[sample + 1] - qvel[sample]) * inv_dt, inv_dt = float32(1 / (timestep * n_substeps))
        computed in double from the model's float32 timestep. Built on the device."""
        t = self.torch
        n = self.lib.locosim_dataset_rows(self.h)
        out = t.empty((n, self.nq), dtype=t.float32, device=self.device)
        self._check(self.lib.locosim_create_dataset_inverse(self.h, _ptr(out), self._stream()))
        self.launches += 1
        return out

    def dynamics_terms(self, M=None, bias=None, passive=None, com=None, jac=None, jac_com=None):
        """Dynamics terms of include/locosim.h (locosim_dynamics_terms) of every env at its stored state and parameter-pool
        row, written into the float32 cuda tensors given (each may be None): M [n_envs, nq, nq] (mj_fullM, armature on the
        diagonal), bias [n_envs, nq] (qfrc_bias), passive [n_envs, nq] (qfrc_passive), com [n_envs, COM_DIM] (whole-robot
        CoM x, y, z, then the total mass), jac [n_envs, nbody, 6, nq] (mj_jacBody at each body's xpos: jacr rows, then
        jacp rows), jac_com [n_envs, 3, nq] (mj_jacSubtreeCom of the robot). The tensors must not overlap. A non-finite
        state gives that env zero rows. Changes nothing else in the engine; stream-ordered, no allocation (can be captured
        in a CUDA graph). Returns {name: tensor} of the outputs given; with none given, launches nothing."""
        n, nq = self.n_envs, self.nq
        outs = (("M", M, (n, nq, nq)), ("bias", bias, (n, nq)), ("passive", passive, (n, nq)), ("com", com, (n, COM_DIM)),
                ("jac", jac, (n, self.nbody, 6, nq)), ("jac_com", jac_com, (n, 3, nq)))
        for name, x, shape in outs:
            if x is not None:
                self._check_tensor(x, name, shape)
        self._check_disjoint(outs)
        given = {name: x for name, x, _ in outs if x is not None}
        if not given:
            return given
        self._check(self.lib.locosim_dynamics_terms(self.h, _ptr(M), _ptr(bias), _ptr(passive), _ptr(com), _ptr(jac),
                                                     _ptr(jac_com), self._stream()))
        self.launches += 1
        return given

    def forward(self, action, dof=None, body_acc=None, cfrc_int=None, cfrc_ext=None):
        """Forward dynamics of include/locosim.h (locosim_forward: one mj_forward, then mj_rnePostConstraint) of every env at
        its stored state, warm start and parameter-pool row under `action` float32 cuda [n_envs, action_dim] (mapped to
        ctrl as a step maps it), with the registered applied forces; written into the float32 cuda tensors given (each may
        be None): dof [n_envs, nq, DOF_DIM] (qfrc_actuator, qfrc_constraint, qacc of this evaluation), body_acc
        [n_envs, nbody, BODY_ACC_DIM] (angular acceleration, linear acceleration of xpos minus gravity), cfrc_int and
        cfrc_ext [n_envs, nbody, CONTACT_DIM] (force, torque about xpos: from the parent through the joints, and external).
        The tensors must not overlap each other or `action`. A non-finite state or action gives that env zero rows. Changes
        nothing in the engine; stream-ordered, no allocation (can be captured in a CUDA graph). Returns {name: tensor} of the
        outputs given; with none given, launches nothing."""
        if action is None:
            raise ValueError("action is required")
        n, nq, nb = self.n_envs, self.nq, self.nbody
        outs = (("action", action, (n, self.action_dim)), ("dof", dof, (n, nq, DOF_DIM)),
                ("body_acc", body_acc, (n, nb, BODY_ACC_DIM)), ("cfrc_int", cfrc_int, (n, nb, CONTACT_DIM)),
                ("cfrc_ext", cfrc_ext, (n, nb, CONTACT_DIM)))
        for name, x, shape in outs:
            if x is not None:
                self._check_tensor(x, name, shape)
        self._check_disjoint(outs)
        given = {name: x for name, x, _ in outs[1:] if x is not None}
        if not given:
            return given
        self._check(self.lib.locosim_forward(self.h, _ptr(action), _ptr(dof), _ptr(body_acc), _ptr(cfrc_int), _ptr(cfrc_ext),
                                             self._stream()))
        self.launches += 1
        return given

    def ray(self, pnt, vec, dist, geom, normal=None, frame=RAY_WORLD, frame_body=0, exclude_body=-1,
            flags=RAY_STATIC | RAY_DYNAMIC):
        """Ray casting of include/locosim.h (locosim_ray, MuJoCo's mj_ray) against every env's geoms at its stored state:
        the rays pnt + x vec, float32 cuda [n_rays, 3] for every env or, with RAY_PER_ENV in `flags`, [n_envs, n_rays, 3],
        given in `frame` (RAY_WORLD, RAY_BODY, RAY_HEADING or RAY_TRACK) of body `frame_body`. Writes dist float32
        [n_envs, n_rays] (the first hit in units of |vec|, -1: none), geom int32 [n_envs, n_rays] (the geom index, -1:
        none) and, when given, normal float32 [n_envs, n_rays, 3] (unit outward normal at the hit, world frame). `flags`
        selects RAY_STATIC (welded to the world: the floor) and / or RAY_DYNAMIC (the robot's) geoms; the geoms of body
        `exclude_body` (-1: none) are skipped. The outputs must not overlap each other or the inputs. Changes nothing in
        the engine; stream-ordered, no allocation (can be captured in a CUDA graph)."""
        n = self.n_envs
        if frame not in (RAY_WORLD, RAY_BODY, RAY_HEADING, RAY_TRACK):
            raise ValueError("unknown ray frame %r" % (frame,))
        if int(flags) & ~(RAY_STATIC | RAY_DYNAMIC | RAY_PER_ENV):
            raise ValueError("unknown ray flag bits in %r" % (flags,))
        if not 0 <= int(frame_body) < self.nbody:
            raise ValueError("frame_body %r out of range [0, %d)" % (frame_body, self.nbody))
        if not -1 <= int(exclude_body) < self.nbody:
            raise ValueError("exclude_body %r out of range [-1, %d)" % (exclude_body, self.nbody))
        shape = getattr(pnt, "shape", None)
        if shape is None or len(shape) < 2:
            raise ValueError("pnt must be a float32 tensor [n_rays, 3] or [n_envs, n_rays, 3]")
        r = int(shape[-2])
        if not 1 <= r <= RAY_MAX:
            raise ValueError("n_rays %d out of range [1, %d]" % (r, RAY_MAX))
        ins = (n, r, 3) if int(flags) & RAY_PER_ENV else (r, 3)
        spans = (("pnt", pnt, ins), ("vec", vec, ins), ("dist", dist, (n, r)), ("geom", geom, (n, r)),
                 ("normal", normal, (n, r, 3)))
        for name, x, shp in spans:
            if x is not None or name != "normal":
                self._check_tensor(x, name, shp, "int32" if name == "geom" else "float32")
        # the inputs may share memory with each other; every output is checked against everything else
        self._check_disjoint(spans[2:] + spans[:1])
        self._check_disjoint(spans[2:] + spans[1:2])
        self._check(self.lib.locosim_ray(self.h, _ptr(pnt), _ptr(vec), r, int(frame), int(frame_body), int(exclude_body),
                                         int(flags), _ptr(dist), _ptr(geom), _ptr(normal), self._stream()))
        self.launches += 1
        return dist, geom, normal

    @property
    def state_layout(self):
        """{field: (offset, length)} of a saved-state row (`state_layout(nq, obs_dim)`)."""
        return state_layout(self.nq, self.obs_dim)

    def save_state(self, obs, out=None):
        """Save every env's whole state (include/locosim.h locosim_save_state): int32 cuda [n_envs, state_words], one row per
        env (`state_layout`), written into `out` (or a new tensor) and returned. `obs` float32 cuda [n_envs, obs_dim] is the
        observation the envs act on next (a step's next_obs, a reset's observation); it is stored in the row. Stream-ordered,
        no allocation when `out` is given (can be captured in a CUDA graph)."""
        t = self.torch
        shape = (self.n_envs, self.state_words)
        if out is None:
            out = t.empty(shape, dtype=t.int32, device=self.device)
        self._check_tensor(obs, "obs", (self.n_envs, self.obs_dim))
        self._check_tensor(out, "out", shape, "int32")
        self._check_disjoint((("obs", obs, (self.n_envs, self.obs_dim)), ("out", out, shape)))
        self._check(self.lib.locosim_save_state(self.h, _ptr(obs), _ptr(out), self._stream()))
        self.launches += 1
        return out

    def load_state(self, rows, index=None, obs_out=None):
        """Load saved states (include/locosim.h locosim_load_state): env i takes row index[i] of `rows` int32 cuda
        [M, state_words] (M >= 1, any size); `index` int32 cuda [n_envs], or None for row i (then M must be n_envs). An env
        whose index is negative or >= M, or whose row comes from an engine of another layout, is left untouched. The stored
        observations of the loaded envs are written into `obs_out` float32 cuda [n_envs, obs_dim] if given (other rows are
        not written). With body or reference outputs registered, their next-state rows of the loaded envs are rewritten
        (one more kernel). Stream-ordered, no allocation (can be captured in a CUDA graph)."""
        n, W, D = self.n_envs, self.state_words, self.obs_dim
        rshape = tuple(getattr(rows, "shape", ()))
        m = rshape[0] if len(rshape) == 2 and rshape[0] >= 1 else 1
        self._check_tensor(rows, "rows", (m, W), "int32")
        spans = [("rows", rows, (m, W))]
        if index is None:
            if m != n:
                raise ValueError("rows must have one row per env (%d) when no index is given, not %d" % (n, m))
        else:
            self._check_tensor(index, "index", (n,), "int32")
            spans.append(("index", index, (n,)))
        if obs_out is not None:
            self._check_tensor(obs_out, "obs_out", (n, D))
            spans.append(("obs_out", obs_out, (n, D)))
        self._check_disjoint(spans)
        self._check(self.lib.locosim_load_state(self.h, _ptr(rows), m, _ptr(index), _ptr(obs_out), self._stream()))
        self.launches += 1 if self._body_out[1] is None and self._ref_out == (None, None) else 2
        return obs_out

    def set_goal(self, goal):
        """goal: float32 cuda [n_envs, 4] per-episode goal features (A1: cos, sin, speed)."""
        self._check_tensor(goal, "goal", (self.n_envs, 4))
        self._check(self.lib.locosim_set_goal(self.h, _ptr(goal), self._stream()))

    def set_param_pool(self, pool):
        """pool: float64 [n_rows, row_len] (domain_randomization.pool_row layout)."""
        pool = np.ascontiguousarray(pool, dtype=np.float64)
        if pool.ndim != 2 or pool.shape[1] != self.lib.locosim_param_pool_row_len(self.h):
            raise ValueError("pool row length %s != %d" % (pool.shape, self.lib.locosim_param_pool_row_len(self.h)))
        self._check(self.lib.locosim_set_param_pool(self.h, pool.ctypes.data, pool.shape[0], pool.shape[1]))

    def param_rows(self):
        t = self.torch
        r = t.empty((self.n_envs,), dtype=t.int32, device=self.device)
        self._check(self.lib.locosim_get_param_rows(self.h, _ptr(r), self._stream()))
        return r

    def counters(self):
        t = self.torch
        c = t.empty((self.n_envs, 8), dtype=t.int32, device=self.device)
        self._check(self.lib.locosim_get_counters(self.h, _ptr(c), self._stream()))
        return c

    def launch_info(self):
        a, b, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        self.lib.locosim_launch_info(self.h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c))
        return dict(warps_per_block=a.value, smem_bytes=b.value, blocks=c.value)
