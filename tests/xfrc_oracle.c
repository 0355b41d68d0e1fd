/*
 * xfrc_oracle.c -- fp64 reference for external body wrenches (mj_data.xfrc_applied).  TEST INFRASTRUCTURE ONLY.
 *
 * The CPU oracle (oracle/mjstep_oracle.c) is compiled into this translation unit unchanged, and the wrench is added on top of
 * its stages, so the oracle every other parity test shares keeps its exact arithmetic.  What is added ([MJ-upstream]
 * engine_passive.c mj_xfrcAccumulate, engine_forward.c mj_fwdAcceleration, engine_io.c mj_resetData):
 *   qfrc_applied = sum_b Jp_b(xipos_b)^T f_b + Jr_b^T t_b      (force at the body's centre of mass, torque, world axes)
 *   qfrc_smooth  = -qfrc_bias + ctrl + qfrc_applied             (qfrc_bias, which the stable-PD controller reads, stays as it is)
 *   mj_resetData (the auto-reset of mj_checkPos / Vel / Acc) zeroes the wrench.
 * The entry points mirror the oracle's orc_forward / orc_step / orc_env_step with the wrench (xfrc[nb*6], robot bodies, row 0 =
 * root) and qfrc_applied[nv] owned by the caller.
 */
#include "../oracle/mjstep_oracle.c"

/* J^T of the wrench about sub_com (the oracle's spatial origin): force vectors [n; f] with n = t + (xipos - sub_com) x f, summed
 * along each body's dof chain like the contact rows of make_constraints */
static void xfrc_accumulate(const OrcModel* m, const OrcData* d, const double* xfrc, double* qfrc_applied) {
  memset(qfrc_applied, 0, 8 * m->nv);
  const double* O = d->sub_com;
  for (int b = 0; b < m->nb; b++) {
    const double* f = xfrc + 6 * b, *t = f + 3;
    double ip[3], r[3], rf[3], w[6];
    mat_vec(ip, d->xmat + 9 * b, m->ipos + 3 * b);
    for (int i = 0; i < 3; i++) r[i] = d->xpos[3 * b + i] + ip[i] - O[i];
    cross(rf, r, f);
    for (int i = 0; i < 3; i++) { w[i] = t[i] + rf[i]; w[3 + i] = f[i]; }
    int dof = m->dofadr[b] + m->dofnum[b] - 1;
    while (dof >= 0) { qfrc_applied[dof] += dot6(d->S + 6 * dof, w); dof = m->dof_parent[dof]; }
  }
}

void orx_forward(const OrcModel* m, OrcData* d, const double* xfrc, double* qfrc_applied) {
  int nv = m->nv;
  position_stage(m, d);
  collision(m, d);
  velocity_stage(m, d);
  make_constraints(m, d);
  xfrc_accumulate(m, d, xfrc, qfrc_applied);
  for (int i = 0; i < nv; i++) d->qfrc_smooth[i] = -d->qfrc_bias[i] + (i >= 6 ? d->ctrl[i - 6] : 0.0) + qfrc_applied[i];
  memcpy(d->qacc_smooth, d->qfrc_smooth, 8 * nv);
  ltdl_solve(m, d->LD, d->qacc_smooth);
  solve_constraints(m, d);
}

static void reset_data_xfrc(const OrcModel* m, OrcData* d, double* xfrc) {
  reset_data(m, d);
  memset(xfrc, 0, 8 * 6 * m->nb);
}

void orx_step(const OrcModel* m, OrcData* d, double* xfrc, double* qfrc_applied) {
  if (any_bad(d->qpos, m->nq)) { d->warn |= 1; reset_data_xfrc(m, d, xfrc); }
  if (any_bad(d->qvel, m->nv)) { d->warn |= 2; reset_data_xfrc(m, d, xfrc); }
  orx_forward(m, d, xfrc, qfrc_applied);
  if (any_bad(d->qacc, m->nv)) { d->warn |= 4; reset_data_xfrc(m, d, xfrc); orx_forward(m, d, xfrc, qfrc_applied); }
  integrate(m, d);
}

int orx_env_step(const OrcModel* m, OrcData* d, const double* action, double* xfrc, double* qfrc_applied, double* obs, double* reward,
                 int* terminated, int* truncated) {
  if (m->cfg.task != SMPLSIM_TASK_NONE && d->cur_t >= d->change_step) reset_task(m, d);
  memcpy(d->prev_root, d->qpos, 24);
  for (int s = 0; s < m->cfg.nsubsteps; s++) {
    orc_compute_torque(m, d, action, d->last_torque);
    memcpy(d->ctrl, d->last_torque, 8 * m->nu);
    orx_step(m, d, xfrc, qfrc_applied);
  }
  d->cur_t += 1;
  int n = orc_compute_observations(m, d, obs);
  *reward = compute_reward(m, d);
  compute_reset(m, d, terminated, truncated);
  return n;
}
