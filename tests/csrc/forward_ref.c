/*
 * Forward dynamics outputs (include/locosim.h locosim_forward: mj_forward + mj_rnePostConstraint) on top of the fp64 CPU
 * oracle -- TEST INFRASTRUCTURE.
 *
 * The oracle (oracle/locosim_ref.c) stays the fixed yardstick; this translation unit compiles in the inverse-dynamics
 * reference (its forward evaluation with ctrl and applied forces) and restates MuJoCo 2.3.7's mj_rnePostConstraint on the
 * oracle's frames, velocities and constraint forces, walking the tree by body_parentid as MuJoCo does:
 *   cacc[0] = (0, -g);  cacc[b] = cacc[parent] + sum over b's dofs of (cdof_dot qvel + cdof qacc)
 *   cfrc_ext[b] = contacts (mj_contactForce in the world frame, - on geom1's body, + on geom2's) + xfrc_applied[b] moved
 *                 from xipos, all as spatial forces (torque, force) about subtree_com[root]
 *   cfrc_int[b] = cinert cacc + cvel x* (cinert cvel) - cfrc_ext, summed from the leaves to the root
 * and converts them to the engine's layout: mj_objectAcceleration at xpos for the body accelerations, force first about
 * xpos for the two wrenches. Built by tests/forward_ref.py into tests/_build.
 */
#include "inverse_ref.c"

/* spatial force (torque, force) about point `from` -> the same force about point `to`: torque + (from - to) x force */
static void force_about(double* res, const double* f, const double* from, const double* to) {
  double r[3] = {from[0] - to[0], from[1] - to[1], from[2] - to[2]}, rxF[3];
  cross3(rxF, r, f + 3);
  for (int k = 0; k < 3; k++) { res[k] = f[k] + rxF[k]; res[3 + k] = f[3 + k]; }
}

/* Forward evaluation at the sim's state with ctrl [nu] and applied forces (xfrc [nb, 6], qfrc [nv]; either may be NULL),
 * then mj_rnePostConstraint. Outputs in the engine's layout (any may be NULL): dof [nv, 3] (qfrc_actuator,
 * qfrc_constraint, qacc), body_acc [nb, 6], cfrc_int [nb, 6], cfrc_ext [nb, 6]; and, for the tests, MuJoCo's own cacc /
 * cfrc_int / cfrc_ext [nb, 6] (spatial, about subtree_com[root], angular / torque first) in raw [nb, 18] (may be NULL).
 * Returns the solver's iteration count. */
int reffwd_forward(RefSim* s, const double* ctrl, const double* xfrc, const double* qfrc, double* dof, double* body_acc,
                   double* cfrc_int, double* cfrc_ext, double* raw) {
  const Model* m = &s->m;
  const int nv = m->nv, nb = m->nb;
  const int it = refinv_forward(s, ctrl, xfrc, qfrc, NULL, NULL);
  static __thread double cacc[MAXBODY][6], fint[MAXBODY][6], fext[MAXBODY][6];
  memset(cacc, 0, sizeof(cacc));
  memset(fext, 0, sizeof(fext));
  for (int k = 0; k < 3; k++) cacc[0][3 + k] = -m->gravity[k];
  for (int b = 1; b < nb; b++) {
    memcpy(cacc[b], cacc[m->body_parentid[b]], sizeof(double) * 6);
    for (int k = 0; k < m->body_jntnum[b]; k++) {
      const int j = m->body_jntadr[b] + k;
      for (int c = 0; c < 6; c++) cacc[b][c] += s->cdof_dot[j][c] * s->qvel[j] + s->cdof[j][c] * s->qacc[j];
    }
  }
  for (int i = 0; i < s->ncon; i++) {
    const Contact* c = &s->con[i];
    double o[16], w[6], t[6];
    ref_get_contact(s, i, o);
    const double* f = o + 10;
    for (int j = 0; j < 3; j++) {
      w[3 + j] = f[0] * c->frame[j] + f[1] * c->frame[3 + j] + f[2] * c->frame[6 + j];
      w[j] = f[3] * c->frame[j] + f[4] * c->frame[3 + j] + f[5] * c->frame[6 + j];
    }
    const int bs[2] = {m->geom_bodyid[c->geom1], m->geom_bodyid[c->geom2]};
    for (int side = 0; side < 2; side++) {
      const int b = bs[side];
      if (b == 0) continue;
      force_about(t, w, c->pos, s->subtree_com[m->body_rootid[b]]);
      for (int k = 0; k < 6; k++) fext[b][k] += side == 1 ? t[k] : -t[k];
    }
  }
  if (xfrc)
    for (int b = 1; b < nb; b++) {
      double w[6] = {xfrc[6 * b + 3], xfrc[6 * b + 4], xfrc[6 * b + 5], xfrc[6 * b], xfrc[6 * b + 1], xfrc[6 * b + 2]}, t[6];
      force_about(t, w, s->xipos[b], s->subtree_com[m->body_rootid[b]]);
      for (int k = 0; k < 6; k++) fext[b][k] += t[k];
    }
  memset(fint, 0, sizeof(fint));
  for (int b = 1; b < nb; b++) {
    double t1[6], t2[6], t3[6];
    mulInertVec(t1, s->cinert[b], cacc[b]);
    mulInertVec(t2, s->cinert[b], s->cvel[b]);
    crossForce(t3, s->cvel[b], t2);
    for (int c = 0; c < 6; c++) fint[b][c] = t1[c] + t3[c] - fext[b][c];
  }
  for (int b = nb - 1; b > 0; b--) {
    const int p = m->body_parentid[b];
    if (p > 0) for (int c = 0; c < 6; c++) fint[p][c] += fint[b][c];
  }
  if (dof)
    for (int d = 0; d < nv; d++) {
      dof[3 * d] = s->qfrc_actuator[d]; dof[3 * d + 1] = s->qfrc_constraint[d]; dof[3 * d + 2] = s->qacc[d];
    }
  for (int b = 0; b < nb; b++) {
    const double* com = s->subtree_com[b > 0 ? m->body_rootid[b] : 0];
    const double r[3] = {s->xpos[b][0] - com[0], s->xpos[b][1] - com[1], s->xpos[b][2] - com[2]};
    if (raw) for (int c = 0; c < 6; c++) { raw[18 * b + c] = cacc[b][c]; raw[18 * b + 6 + c] = fint[b][c]; raw[18 * b + 12 + c] = fext[b][c]; }
    if (body_acc) {
      /* mj_objectAcceleration(mjOBJ_XBODY, flg_local = 0): acceleration and velocity moved to xpos, plus w x v */
      const double* w = s->cvel[b];
      double ar[3], wr[3], vp[3], wv[3];
      cross3(ar, cacc[b], r);
      cross3(wr, w, r);
      for (int k = 0; k < 3; k++) vp[k] = w[3 + k] + wr[k];
      cross3(wv, w, vp);
      for (int k = 0; k < 3; k++) { body_acc[6 * b + k] = cacc[b][k]; body_acc[6 * b + 3 + k] = cacc[b][3 + k] + ar[k] + wv[k]; }
    }
    double t[6];
    if (cfrc_int) {
      force_about(t, fint[b], com, s->xpos[b]);
      for (int k = 0; k < 3; k++) { cfrc_int[6 * b + k] = t[3 + k]; cfrc_int[6 * b + 3 + k] = t[k]; }
    }
    if (cfrc_ext) {
      force_about(t, fext[b], com, s->xpos[b]);
      for (int k = 0; k < 3; k++) { cfrc_ext[6 * b + k] = t[3 + k]; cfrc_ext[6 * b + 3 + k] = t[k]; }
    }
  }
  return it;
}

/* for the tests' identities: cdof [nv, 6], cinert [nb, 10], xipos [nb, 3], subtree_com of every body [nb, 3] and the
 * passive force [nv] of the last evaluation (any may be NULL) */
void reffwd_frames(const RefSim* s, double* cdof, double* cinert, double* xipos, double* subtree_com, double* passive) {
  const Model* m = &s->m;
  for (int j = 0; j < m->nv; j++) {
    if (cdof) for (int c = 0; c < 6; c++) cdof[6 * j + c] = s->cdof[j][c];
    if (passive) passive[j] = s->qfrc_passive[j];
  }
  for (int b = 0; b < m->nb; b++) {
    if (cinert) for (int c = 0; c < 10; c++) cinert[10 * b + c] = s->cinert[b][c];
    for (int c = 0; c < 3; c++) {
      if (xipos) xipos[3 * b + c] = s->xipos[b][c];
      if (subtree_com) subtree_com[3 * b + c] = s->subtree_com[b][c];
    }
  }
}

/* the oracle's kinematics and com_pos stages alone at qpos: xpos [nb, 3], cdof [nv, 6] and subtree_com [nb, 3] (any may be
 * NULL), for the body Jacobians and their central differences along qvel */
void reffwd_kin(RefSim* s, const double* qpos, double* xpos, double* cdof, double* subtree_com) {
  memcpy(s->qpos, qpos, sizeof(double) * s->m.nv);
  kinematics(s);
  comPos(s);
  for (int b = 0; b < s->m.nb; b++)
    for (int k = 0; k < 3; k++) {
      if (xpos) xpos[3 * b + k] = s->xpos[b][k];
      if (subtree_com) subtree_com[3 * b + k] = s->subtree_com[b][k];
    }
  for (int j = 0; j < s->m.nv; j++) if (cdof) for (int c = 0; c < 6; c++) cdof[6 * j + c] = s->cdof[j][c];
}
