"""fp64 reference of the contact list (include/locosim.h locosim_set_contact_list_outputs) and its comparison with the engine's
rows -- TEST INFRASTRUCTURE ONLY (never imported by the package). The reference is the oracle's contact list of its last
forward evaluation (tests/contact_wrench_ref.py: refcw_get_contact), less the contacts MuJoCo keeps without a constraint
(dist >= margin - gap), which the engine leaves out of its list."""
import ctypes

import numpy as np

import contact_wrench_ref as cwr

DIM, ID_DIM = 19, 5          # LS_CONLIST_DIM, LS_CONLIST_ID_DIM
# Tolerances of the fp32 engine against the fp64 reference after one control step from the same state: dist and pos 2 mm,
# frame components 2e-3, forces 2 N (the contact-wrench tests' TOL; the torsional and rolling components are N m)
TOL = dict(dist=2e-3, pos=2e-3, frame=2e-3, force=2.0)


def reference(o, sim, model):
    """the reference list of the oracle sim's last forward evaluation: dict of numpy arrays in list order (dist [n], pos
    [n, 3], frame [n, 9], force [n, 6], geom [n, 2], body [n, 2], dim [n])"""
    rows = cwr.contacts(o, sim)
    if len(rows):
        g1, g2 = rows[:, 13].astype(int), rows[:, 14].astype(int)
        incl = np.maximum(model.geom_margin[g1], model.geom_margin[g2]) - np.maximum(model.geom_gap[g1], model.geom_gap[g2])
        rows = rows[rows[:, 0] < incl]
    geom = rows[:, 13:15].astype(np.int64)
    return dict(dist=rows[:, 0], pos=rows[:, 1:4], frame=rows[:, 4:13], force=rows[:, 16:22], geom=geom,
                body=np.asarray(model.geom_bodyid)[geom].reshape(-1, 2), dim=rows[:, 15].astype(np.int64))


def unpack(ncon, con, con_id):
    """one env's engine rows (ncon int, con [C, DIM], con_id [C, ID_DIM], numpy) -> the reference's dict, first ncon rows"""
    n = int(ncon)
    c, i = np.asarray(con, dtype=np.float64)[:n], np.asarray(con_id)[:n].astype(np.int64)
    return dict(dist=c[:, 0], pos=c[:, 1:4], frame=c[:, 4:13], force=c[:, 13:19], geom=i[:, 0:2], body=i[:, 2:4],
                dim=i[:, 4])


def mismatch(got, want):
    """how far the engine's list is from the reference: inf when the contacts differ (count, geom pairs or dim, in list
    order), else the largest error of any field relative to its tolerance (<= 1: within TOL)"""
    if len(got["dist"]) != len(want["dist"]) or not np.array_equal(got["geom"], want["geom"]) \
            or not np.array_equal(got["dim"], want["dim"]) or not np.array_equal(got["body"], want["body"]):
        return np.inf
    if len(got["dist"]) == 0:
        return 0.0
    return max(float(np.abs(got[k] - want[k]).max()) / TOL[k] for k in TOL)


def empty_rows_ok(ncon, con, con_id):
    """rows at and past ncon hold exact zeros and ids of -1"""
    n = int(ncon)
    return bool(np.all(np.asarray(con)[n:] == 0) and np.all(np.asarray(con_id)[n:] == -1))


def sensitivity(o, model_blobs, task_blobs, model, qpos, qvel, action, want, warmstart=None, eps=1e-6, n_probe=8, seed=0,
                user=None):
    """How far the ORACLE's own list moves (mismatch against `want`) when its start state is perturbed by `eps` (fp32
    resolution): where a contact switches on or off within the step, the list is discontinuous and an fp32 engine may take
    the other branch (inf: the perturbed oracle itself has another list)."""
    rng = np.random.RandomState(seed)
    gap = 0.0
    for _ in range(n_probe):
        oe = o.env(model_blobs, task_blobs)
        if user is not None:
            oe.set_user(user)
        oe.set_state(qpos + eps * rng.randn(len(qpos)), qvel + eps * rng.randn(len(qvel)), warmstart)
        cwr.env_step(o, oe, action)
        gap = max(gap, mismatch(reference(o, oe.sim, model), want))
        oe.close()
    return gap


def emu_bind(emu):
    """declare emu_set_contact_list(sim, ncon int32 [1], con fp32 [C, DIM], con_id int32 [C, ID_DIM] | all NULL) and
    emu_max_contacts(sim) on the emulation library"""
    emu.emu_set_contact_list.restype = None
    emu.emu_set_contact_list.argtypes = [ctypes.c_void_p] * 4
    emu.emu_max_contacts.restype = ctypes.c_int
    emu.emu_max_contacts.argtypes = [ctypes.c_void_p]
    return emu
