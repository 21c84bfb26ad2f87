"""fp64 reference of the reference outputs (include/locosim.h locosim_set_reference_outputs) and the serial emulation build's
entry point for one reference row -- TEST INFRASTRUCTURE ONLY (never imported by the package).

A reference row is the body-output row (tests/body_outputs_ref.BodyRef) of the reset state of one row of the reset table:
root x / y zeroed and, under setup_random_rot, the yaw shifted by the angle (wrapped to [-pi, pi)) and root (vx, vy) rotated
by it (locosim_core.cuh reset_value; unitreeA1.py setup_random_rot)."""
import ctypes

import numpy as np

from body_outputs_ref import BODY_DIM, _p


def reset_state(spec, row, nv, angle):
    """fp64 (qpos, qvel) of a reset onto table row `row` ([2 nv + n_goal]) under rotation `angle` (TaskSpec `spec`)."""
    row = np.asarray(row, dtype=np.float64)
    q, v = row[:nv].copy(), row[nv:2 * nv].copy()
    q[spec.recenter[0]] = 0.0
    q[spec.recenter[1]] = 0.0
    yaw, ivx, ivy = spec.random_rot
    if yaw >= 0:
        q[yaw] = np.mod(q[yaw] + angle + np.pi, 2 * np.pi) - np.pi
        c, s = np.cos(angle), np.sin(angle)
        vx, vy = v[ivx], v[ivy]
        v[ivx], v[ivy] = c * vx - s * vy, s * vx + c * vy
    return q, v


def emu_bind(emu):
    emu.emu_reference_row.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float,
                                      ctypes.c_void_p]
    emu.emu_reference_row.restype = None


def emu_reference_row(emu, sim, spec, row, nb, angle):
    """fp32 [nb, BODY_DIM]: the serial core's reference row of table row `row` (taken in fp32, as the engine holds the table)."""
    row = np.ascontiguousarray(row, dtype=np.float32)
    recenter = np.ascontiguousarray(spec.recenter, dtype=np.int32)
    rot = np.ascontiguousarray(spec.random_rot, dtype=np.int32)
    out = np.zeros((nb, BODY_DIM), dtype=np.float32)
    emu.emu_reference_row(sim, _p(row), _p(recenter), _p(rot), float(angle), _p(out))
    return out
