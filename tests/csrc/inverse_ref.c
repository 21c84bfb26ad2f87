/*
 * Inverse dynamics (include/locosim.h locosim_inverse, MuJoCo 2.3.7's continuous-time mj_inverse) on top of the fp64 CPU
 * oracle -- TEST INFRASTRUCTURE.
 *
 * The oracle (oracle/locosim_ref.c) stays the fixed yardstick; this translation unit compiles it in (through the applied-
 * forces reference, for forward solutions with qfrc_applied / xfrc_applied) and composes its own stages. A forward
 * evaluation at the state leaves M (with armature), qfrc_bias, qfrc_passive, the constraint rows J, efc_D and efc_aref
 * behind; the acceleration stage of mj_inverse (mj_invConstraint) is then the oracle's constraint_update of
 * jar = J qacc - aref, followed by mulJT and mulM:
 *   qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - J^T efc_force
 * Built by tests/inverse_ref.py into tests/_build.
 */
#include "applied_forces_ref.c"

/* forward evaluation at the sim's state with ctrl and applied forces (either may be NULL): qacc, qfrc_actuator [nv] out
 * (either may be NULL); returns the solver's iteration count */
int refinv_forward(RefSim* s, const double* ctrl, const double* xfrc, const double* qfrc, double* qacc, double* actuator) {
  if (ctrl) memcpy(s->ctrl, ctrl, sizeof(double) * s->m.nu);
  forward_applied(s, xfrc, qfrc);
  if (qacc) memcpy(qacc, s->qacc, sizeof(double) * s->m.nv);
  if (actuator) memcpy(actuator, s->qfrc_actuator, sizeof(double) * s->m.nv);
  return s->solver_iter;
}

/* mj_inverse at the sim's state (the rows of its last forward evaluation) and qacc [nv]: qfrc_inverse [nv] into out,
 * qfrc_constraint [nv] into cons (may be NULL) and, per dof, the first-order fp32 error scale (may be NULL)
 *   S_d = sum_j |M_dj qacc_j| + |bias_d| + |passive_d| + sum_r |J_rd| (|f_r| + D_r (sum_j |J_rj qacc_j| + |aref_r|))
 * Returns the constraint cost of qacc. The solver's own efc_force is overwritten. */
double refinv_inverse(RefSim* s, const double* qacc, double* out, double* cons, double* scale) {
  const int nv = s->m.nv, n = s->nefc;
  static __thread double jar[MAXEFC], jabs[MAXEFC];
  double Ma[MAXNV], qc[MAXNV];
  for (int i = 0; i < n; i++) {
    double a = 0, b = 0;
    for (int d = 0; d < nv; d++) { a += s->J[i][d] * qacc[d]; b += fabs(s->J[i][d] * qacc[d]); }
    jar[i] = a - s->efc_aref[i];
    jabs[i] = b + fabs(s->efc_aref[i]);
  }
  const double cost = constraint_update(s, jar, NULL, 1);
  mulJT(s, qc, s->efc_force);
  mulM(s, Ma, qacc);
  for (int d = 0; d < nv; d++) {
    out[d] = Ma[d] + s->qfrc_bias[d] - s->qfrc_passive[d] - qc[d];
    if (cons) cons[d] = qc[d];
    if (!scale) continue;
    double sd = fabs(s->qfrc_bias[d]) + fabs(s->qfrc_passive[d]);
    for (int j = 0; j < nv; j++) sd += fabs(s->M[d][j] * qacc[j]);
    for (int i = 0; i < n; i++) sd += fabs(s->J[i][d]) * (fabs(s->efc_force[i]) + s->efc_D[i] * jabs[i]);
    scale[d] = sd;
  }
  return cost;
}

/* the Newton solver's cost at qacc [nv] over the rows of the last forward evaluation: the Gauss term
 * 0.5 (M qacc - qfrc_smooth) . (qacc - qacc_smooth) plus the constraint cost (the cost whose gradient is
 * M qacc - qfrc_smooth - J^T efc_force) */
double refinv_cost(RefSim* s, const double* qacc) {
  const int nv = s->m.nv, n = s->nefc;
  static __thread double jar[MAXEFC];
  double Ma[MAXNV], g = 0;
  for (int i = 0; i < n; i++) {
    double a = 0;
    for (int d = 0; d < nv; d++) a += s->J[i][d] * qacc[d];
    jar[i] = a - s->efc_aref[i];
  }
  mulM(s, Ma, qacc);
  for (int d = 0; d < nv; d++) g += 0.5 * (Ma[d] - s->qfrc_smooth[d]) * (qacc[d] - s->qacc_smooth[d]);
  return g + constraint_update(s, jar, NULL, 0);
}

/* meaninertia of the model (the solver's scale = 1 / (meaninertia * nv)) */
double refinv_meaninertia(const RefSim* s) { return s->m.meaninertia; }
