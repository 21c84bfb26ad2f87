/*
 * Per-dof outputs (include/locosim.h locosim_set_dof_outputs) on top of the fp64 CPU oracle -- TEST INFRASTRUCTURE.
 *
 * The oracle (oracle/locosim_ref.c) stays the fixed yardstick of the physics it already covers; this translation unit
 * compiles it in and reads what its forward evaluation leaves behind, as MuJoCo's mjData holds it:
 *   qfrc_actuator    mj_fwdActuation: gear * force per actuator (ctrlrange, then gain / bias, then forcerange), summed per dof;
 *   qfrc_constraint  J^T efc_force at the solver's final qacc (mj_fwdConstraint);
 *   qacc             the constrained acceleration (mj_forward; the Euler integrator's implicit-damping solve is not stored);
 * and the window of the engine's output: the mean over a control step's sub-steps, each sub-step's values taken after it
 * (its last dynamics evaluation: Euler's only one, RK4's fourth stage).
 * Built by tests/dof_outputs_ref.py into tests/_build.
 */
#include "../../oracle/locosim_ref.c"

#define DOF_DIM 3

/* [nv, 3] (qfrc_actuator, qfrc_constraint, qacc) of the last forward evaluation, ADDED to out */
void refdof_add(const RefSim* s, double* out) {
  for (int d = 0; d < s->m.nv; d++) {
    out[DOF_DIM * d] += s->qfrc_actuator[d];
    out[DOF_DIM * d + 1] += s->qfrc_constraint[d];
    out[DOF_DIM * d + 2] += s->qacc[d];
  }
}

/* qfrc_passive and qfrc_actuator [nv] of the last forward evaluation (the parts of qfrc_smooth, with - qfrc_bias) */
void refdof_get_forces(const RefSim* s, double* passive, double* actuator) {
  memcpy(passive, s->qfrc_passive, sizeof(double) * s->m.nv);
  memcpy(actuator, s->qfrc_actuator, sizeof(double) * s->m.nv);
}

/* nsub sub-steps of a bare RefSim at ctrl, and the mean [nv, 3] over them */
void refdof_step(RefSim* s, const double* ctrl, int nsub, double* out) {
  memset(out, 0, sizeof(double) * DOF_DIM * s->m.nv);
  for (int k = 0; k < nsub; k++) {
    ref_step(s, ctrl, 1);
    refdof_add(s, out);
  }
  for (int j = 0; j < DOF_DIM * s->m.nv; j++) out[j] /= nsub;
}

/* the physics of one control step of a RefEnv (action in [-1, 1] -> ctrl as refenv_step maps it, n_substeps sub-steps of
 * ref_step) and the mean [nv, 3] over its sub-steps; observation, reward and termination are not evaluated */
void refdof_env_step(RefEnv* e, const double* action, double* out) {
  const Task* t = &e->task;
  RefSim* s = e->sim;
  double ctrl[MAXNV];
  memset(ctrl, 0, sizeof(ctrl));
  for (int i = 0; i < s->m.nu; i++) ctrl[t->act_idx[i]] = action[i] * t->act_delta[i] + t->act_mean[i];
  refdof_step(s, ctrl, t->n_substeps, out);
}
