/*
 * Dynamics terms (include/locosim.h locosim_dynamics_terms) on top of the fp64 CPU oracle -- TEST INFRASTRUCTURE.
 *
 * The oracle (oracle/locosim_ref.c) stays the fixed yardstick; this translation unit compiles it in and reads its stages:
 * M (mj_fullM, armature included), qfrc_bias and qfrc_passive after a forward evaluation at the state, and the kinematics
 * alone (xpos, xquat, xipos) for the centre of mass and for the central differences of tests/dynamics_terms_ref.py. It
 * also returns the first-order fp32 error scales of M and qfrc_bias: the sums of the absolute values of the products the
 * oracle's own passes add up (crb, rne_bias), on the magnitudes of their factors (mag_vec, mag_inert), so that neither a
 * cancellation in the result nor a zero of the model's structure shrinks its bound.
 * Built by tests/dynamics_terms_ref.py into tests/_build.
 */
#include "../../oracle/locosim_ref.c"

int refdyn_nbody(const RefSim* s) { return s->m.nb; }

/* Magnitudes of a spatial vector's angular and linear parts, and of a com-frame inertia's rotational, moment and mass
 * parts, broadcast over their entries: an entry that is zero in fp64 because of the model's structure (an axis along a world
 * axis, a planar chain) is a rounding of that part's size in fp32, so every entry is bounded by its part's magnitude */
static void mag_vec(double* r, const double* v) {
  const double a = fmax(fabs(v[0]), fmax(fabs(v[1]), fabs(v[2]))), l = fmax(fabs(v[3]), fmax(fabs(v[4]), fabs(v[5])));
  for (int k = 0; k < 3; k++) { r[k] = a; r[3 + k] = l; }
}
static void mag_inert(double* r, const double* i) {
  double a = 0, h = 0;
  for (int k = 0; k < 6; k++) a = fmax(a, fabs(i[k]));
  for (int k = 6; k < 9; k++) h = fmax(h, fabs(i[k]));
  for (int k = 0; k < 6; k++) r[k] = a;
  for (int k = 6; k < 9; k++) r[k] = h;
  r[9] = fabs(i[9]);
}
/* |I| |v| of mulInertVec, every product counted with its absolute value, on the magnitudes above */
static void abs_inert_vec(double* r, const double* i_, const double* v) {
  double a[10], w[6];
  mag_inert(a, i_);
  mag_vec(w, v);
  r[0] = a[0] * w[0] + a[3] * w[1] + a[4] * w[2] + a[8] * w[4] + a[7] * w[5];
  r[1] = a[3] * w[0] + a[1] * w[1] + a[5] * w[2] + a[8] * w[3] + a[6] * w[5];
  r[2] = a[4] * w[0] + a[5] * w[1] + a[2] * w[2] + a[7] * w[3] + a[6] * w[4];
  r[3] = a[8] * w[1] + a[7] * w[2] + a[9] * w[3];
  r[4] = a[6] * w[2] + a[8] * w[0] + a[9] * w[4];
  r[5] = a[7] * w[0] + a[6] * w[1] + a[9] * w[5];
}
/* |a| x |b| with both products of each component added */
static void abs_cross(double* r, const double* a, const double* b) {
  r[0] = fabs(a[1] * b[2]) + fabs(a[2] * b[1]);
  r[1] = fabs(a[2] * b[0]) + fabs(a[0] * b[2]);
  r[2] = fabs(a[0] * b[1]) + fabs(a[1] * b[0]);
}

/* Forward evaluation at (qpos, qvel) with zero controls, then: M [nv, nv], bias [nv], passive [nv], com [4] (x, y, z of
 * sum m_b xipos_b / sum m_b, then sum m_b), and the error scales sM [nv, nv], sbias [nv] (any output may be NULL) */
void refdyn_terms(RefSim* s, const double* qpos, const double* qvel, double* M, double* bias, double* passive, double* com,
                  double* sM, double* sbias) {
  const Model* m = &s->m;
  const int nv = m->nv, nb = m->nb;
  ref_reset(s, qpos, qvel);
  ref_forward(s, NULL);
  if (M) ref_get_M(s, M);
  if (bias) ref_get_bias(s, bias);
  if (passive) memcpy(passive, s->qfrc_passive, sizeof(double) * nv);
  if (com) {
    double sm = 0, c[3] = {0, 0, 0};
    for (int b = 0; b < nb; b++) {
      sm += m->body_mass[b];
      for (int k = 0; k < 3; k++) c[k] += m->body_mass[b] * s->xipos[b][k];
    }
    for (int k = 0; k < 3; k++) com[k] = c[k] / sm;
    com[3] = sm;
  }
  if (sM) {
    for (int i = 0; i < nv * nv; i++) sM[i] = 0;
    for (int i = 0; i < nv; i++) {
      double buf[6];
      abs_inert_vec(buf, s->crb[m->jnt_bodyid[i]], s->cdof[i]);
      for (int j = i; j >= 0; j = m->dof_parentid[j]) {
        double v = 0, cj[6];
        mag_vec(cj, s->cdof[j]);
        for (int k = 0; k < 6; k++) v += cj[k] * buf[k];
        if (j == i) v += fabs(m->dof_armature[i]);
        sM[i * nv + j] = sM[j * nv + i] = v;
      }
    }
  }
  if (sbias) {
    /* per body |I a| + |v x* (I v)| with the oracle's cacc / cvel, summed over each dof's subtree, against |cdof| */
    static __thread double f[MAXBODY][6];
    memset(f, 0, sizeof(f));
    for (int b = 1; b < nb; b++) {
      double t1[6], t2[6], a3[3], b3[3], c3[3], cv[6];
      abs_inert_vec(t1, s->cinert[b], s->cacc[b]);
      abs_inert_vec(t2, s->cinert[b], s->cvel[b]);
      mag_vec(cv, s->cvel[b]);
      abs_cross(a3, cv, t2);
      abs_cross(b3, cv + 3, t2 + 3);
      abs_cross(c3, cv, t2 + 3);
      for (int k = 0; k < 3; k++) { f[b][k] = t1[k] + a3[k] + b3[k]; f[b][3 + k] = t1[3 + k] + c3[k]; }
    }
    for (int b = nb - 1; b > 0; b--)
      for (int c = 0; c < 6; c++) f[m->body_parentid[b]][c] += f[b][c];
    for (int j = 0; j < nv; j++) {
      double v = 0, cj[6];
      mag_vec(cj, s->cdof[j]);
      for (int c = 0; c < 6; c++) v += cj[c] * f[m->jnt_bodyid[j]][c];
      sbias[j] = v;
    }
  }
}

/* the oracle's kinematics alone at qpos: xpos [nb, 3], xquat [nb, 4], xipos [nb, 3] (any may be NULL) */
void refdyn_frames(RefSim* s, const double* qpos, double* xpos, double* xquat, double* xipos) {
  const int nb = s->m.nb;
  memcpy(s->qpos, qpos, sizeof(double) * s->m.nv);
  kinematics(s);
  for (int b = 0; b < nb; b++) {
    for (int k = 0; k < 3; k++) {
      if (xpos) xpos[3 * b + k] = s->xpos[b][k];
      if (xipos) xipos[3 * b + k] = s->xipos[b][k];
    }
    if (xquat) for (int k = 0; k < 4; k++) xquat[4 * b + k] = s->xquat[b][k];
  }
}
