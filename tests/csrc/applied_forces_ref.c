/*
 * Applied forces (MuJoCo 2.3.7 mjData.xfrc_applied / qfrc_applied) on top of the fp64 CPU oracle -- TEST INFRASTRUCTURE.
 *
 * The oracle (oracle/locosim_ref.c) stays the fixed yardstick of the physics it already covers; this translation unit
 * compiles it in and adds the two inputs around its stages, restating the documented MuJoCo computation:
 *   mj_fwdAcceleration: qfrc_smooth = qfrc_passive - qfrc_bias + qfrc_actuator + qfrc_applied
 *   mj_xfrcAccumulate:  qfrc_smooth += sum over bodies b >= 1 of J_b^T (force, torque), applied at xipos[b] (mj_applyFT)
 * in every dynamics evaluation (Euler: mj_forward of each sub-step; RK4: each stage), so the solver sees them through
 * qacc_smooth and the implicit-damping Euler step through qfrc_smooth. Everything else is the oracle's own code.
 * Built by tests/applied_forces_ref.py into tests/_build.
 */
#include "../../oracle/locosim_ref.c"

int refx_nbody(const RefSim* s) { return s->m.nb; }

/* qfrc += J^T xfrc: every wrench as a spatial force about the subtree CoM of its root (the frame of cdof), summed over each
 * dof's subtree, projected on cdof */
static void xfrc_accumulate(const RefSim* s, const double* xfrc, double* qfrc) {
  const Model* m = &s->m;
  double f[MAXBODY][6];
  memset(f, 0, sizeof(f));
  for (int b = 1; b < m->nb; b++) {
    const double* w = xfrc + 6 * b;
    const double* com = s->subtree_com[m->body_rootid[b]];
    double r[3] = {s->xipos[b][0] - com[0], s->xipos[b][1] - com[1], s->xipos[b][2] - com[2]}, rxF[3];
    cross3(rxF, r, w);
    for (int k = 0; k < 3; k++) { f[b][k] = w[3 + k] + rxF[k]; f[b][3 + k] = w[k]; }
  }
  for (int b = m->nb - 1; b > 0; b--) {
    int p = m->body_parentid[b];
    for (int k = 0; k < 6; k++) f[p][k] += f[b][k];
  }
  for (int j = 0; j < m->nv; j++) {
    double v = 0;
    for (int k = 0; k < 6; k++) v += s->cdof[j][k] * f[m->jnt_bodyid[j]][k];
    qfrc[j] += v;
  }
}

/* the oracle's forward() with the applied forces added to qfrc_smooth; xfrc [nb, 6] / qfrc [nv] may be NULL */
static void forward_applied(RefSim* s, const double* xfrc, const double* qfrc) {
  const Model* m = &s->m;
  int nv = m->nv;
  kinematics(s);
  comPos(s);
  crb(s);
  collision(s);
  make_constraint(s);
  comVel(s);
  passive(s);
  reference_constraint(s);
  rne_bias(s);
  actuation(s);
  for (int i = 0; i < nv; i++) {
    s->qfrc_smooth[i] = s->qfrc_passive[i] - s->qfrc_bias[i] + s->qfrc_actuator[i];
    if (qfrc) s->qfrc_smooth[i] += qfrc[i];
  }
  if (xfrc) xfrc_accumulate(s, xfrc, s->qfrc_smooth);
  for (int i = 0; i < nv; i++) s->qacc_smooth[i] = s->qfrc_smooth[i];
  chol_solve(s->LM, nv, s->qacc_smooth);
  fwd_constraint(s);
}

/* the oracle's rk4() with forward_applied in its stages */
static void rk4_applied(RefSim* s, const double* xfrc, const double* qfrc) {
  const Model* m = &s->m;
  int nv = m->nv;
  double h = m->timestep;
  static const double A[3][3] = {{0.5, 0, 0}, {0, 0.5, 0}, {0, 0, 1}};
  static const double B[4] = {1.0 / 6, 1.0 / 3, 1.0 / 3, 1.0 / 6};
  double X0q[MAXNV], X0v[MAXNV], Fv[4][MAXNV], Fa[4][MAXNV];
  memcpy(X0q, s->qpos, sizeof(double) * nv);
  memcpy(X0v, s->qvel, sizeof(double) * nv);
  memcpy(Fv[0], s->qvel, sizeof(double) * nv);
  memcpy(Fa[0], s->qacc, sizeof(double) * nv);
  for (int i = 1; i < 4; i++) {
    for (int d = 0; d < nv; d++) {
      double dq = 0, dv = 0;
      for (int j = 0; j < i; j++) { dq += A[i - 1][j] * Fv[j][d]; dv += A[i - 1][j] * Fa[j][d]; }
      s->qpos[d] = X0q[d] + h * dq;
      s->qvel[d] = X0v[d] + h * dv;
    }
    forward_applied(s, xfrc, qfrc);
    memcpy(Fv[i], s->qvel, sizeof(double) * nv);
    memcpy(Fa[i], s->qacc, sizeof(double) * nv);
  }
  for (int d = 0; d < nv; d++) {
    double dq = 0, dv = 0;
    for (int j = 0; j < 4; j++) { dq += B[j] * Fv[j][d]; dv += B[j] * Fa[j][d]; }
    s->qvel[d] = X0v[d] + h * dv;
    s->qpos[d] = X0q[d] + h * dq;
  }
}

/* ref_forward / ref_step with applied forces */
void refx_forward(RefSim* s, const double* ctrl, const double* xfrc, const double* qfrc) {
  if (ctrl) memcpy(s->ctrl, ctrl, sizeof(double) * s->m.nu);
  forward_applied(s, xfrc, qfrc);
}
void refx_step(RefSim* s, const double* ctrl, int nsub, const double* xfrc, const double* qfrc) {
  if (ctrl) memcpy(s->ctrl, ctrl, sizeof(double) * s->m.nu);
  for (int k = 0; k < nsub; k++) {
    forward_applied(s, xfrc, qfrc);
    if (s->m.integrator == 1) rk4_applied(s, xfrc, qfrc); else euler(s);
  }
}

/* the physics of one control step of a RefEnv (action in [-1, 1] -> ctrl as refenv_step maps it, n_substeps sub-steps);
 * observation, reward and termination are not evaluated: compare the state (ref_get_state) */
void refx_env_step(RefEnv* e, const double* action, const double* xfrc, const double* qfrc) {
  const Task* t = &e->task;
  double ctrl[MAXNV];
  memset(ctrl, 0, sizeof(ctrl));
  for (int i = 0; i < e->sim->m.nu; i++) ctrl[t->act_idx[i]] = action[i] * t->act_delta[i] + t->act_mean[i];
  refx_step(e->sim, ctrl, t->n_substeps, xfrc, qfrc);
}

/* body frames of the last forward evaluation: xipos [nb, 3] (centre of mass), xmat [nb, 9] (orientation, row major) */
void refx_get_bodies(const RefSim* s, double* xipos, double* xmat) {
  for (int b = 0; b < s->m.nb; b++) {
    if (xipos) for (int k = 0; k < 3; k++) xipos[3 * b + k] = s->xipos[b][k];
    if (xmat) for (int k = 0; k < 9; k++) xmat[9 * b + k] = s->xmat[b][k];
  }
}
