/* tests/emu/delay_oracle.c — TEST HARNESS ONLY.  The oracle's control step with an action delay (DESIGN.md §7.9), for
 * tests/test_action_delay.py.  It compiles oracle/sim_oracle.c unchanged and restates its orc_step / orc_step_autoreset with one
 * change: substeps s < delay of a control step drive the PD loop towards e->prev_action (the previous control step's target)
 * instead of this step's target.  At delay 0 it is orc_step_autoreset bit for bit, which the tests check; everything else (the
 * physics, the task, the rewards, the resets) is the oracle's own code.  Only delay_oracle_step is exported. */
#include "../../oracle/sim_oracle.c"

static void delay_orc_step(const orc_model* m, orc_env* e, const double* action, int delay, double* obs, double* rew_terms,
                           double* reward, int* done) {
  int nu = m->nu;
  double target[ORC_NU], ctrl[ORC_NU], t[ORC_NREW];
  /* base_humanoid_env.py:209-212 smoothing + nominal offsets ; robot_base.py:80 */
  for (int u = 0; u < nu; u++)
    target[u] = m->action_smoothing * action[u] + (1 - m->action_smoothing) * e->prev_prediction[u] + m->nominal_qpos[7 + u];
  if (!e->have_prev) { /* robot_base.py:82-85 */
    memcpy(e->prev_action, target, sizeof(target));
    memcpy(e->prev_torque, e->act_force, sizeof(e->prev_torque));
    e->have_prev = 1;
  }
  e->rng_ctr++;   /* one event counter per control step; every draw of this step is keyed by it */
  double kp[ORC_NU], kd[ORC_NU];
  memcpy(kp, m->kp, sizeof(kp));
  memcpy(kd, m->kd, sizeof(kd));
  if (m->pdrand_k > 0) {
    /* RobotBase._do_simulation (robots/robot_base.py:41-47): kp ~ U((1-k) kp, (1+k) kp), then kd likewise, once per
     * control step.  joint u -> stream 8 + u/4 (kp) / 11 + u/4 (kd), lane u%4 */
    uint32_t w[4];
    for (int u = 0; u < nu; u++) {
      if ((u & 3) == 0) orc_philox(e->seed, e->env_id, e->rng_ctr, 8 + (u >> 2), w);
      double lo = (1 - m->pdrand_k) * m->kp[u], hi = (1 + m->pdrand_k) * m->kp[u];
      kp[u] = lo + (hi - lo) * u01(w[u & 3]);
    }
    for (int u = 0; u < nu; u++) {
      if ((u & 3) == 0) orc_philox(e->seed, e->env_id, e->rng_ctr, 11 + (u >> 2), w);
      double lo = (1 - m->pdrand_k) * m->kd[u], hi = (1 + m->pdrand_k) * m->kd[u];
      kd[u] = lo + (hi - lo) * u01(w[u & 3]);
    }
  }
  for (int s = 0; s < m->frame_skip; s++) {
    const double* tg = s < delay ? e->prev_action : target;   /* the one change: the first `delay` substeps keep the old target */
    for (int u = 0; u < nu; u++) ctrl[u] = kp[u] * (tg[u] - e->act_len[u]) + kd[u] * (0.0 - e->act_vel[u]);
    orc_mj_step(m, e, ctrl);
  }
  task_step(m, e);
  if (m->task == ORC_TASK_STAND) calc_reward_stand(m, e, t);
  else if (m->task == ORC_TASK_STEP) calc_reward_step(m, e, t);
  else calc_reward(m, e, target, t);
  int d = (e->qpos[2] < m->done_lo) || (e->qpos[2] > m->done_hi) || e->self_collision || e->status;
  if (m->task == ORC_TASK_STEP) {   /* SteppingTask.done (stepping_task.py:248-260): root height above the lower foot site */
    double fz = e->site_pos[0][2] < e->site_pos[1][2] ? e->site_pos[0][2] : e->site_pos[1][2];
    d = (e->root_xpos[2] - fz < m->done_lo) || e->self_collision || e->status;
  }
  memcpy(e->prev_action, target, sizeof(target));
  memcpy(e->prev_torque, e->act_force, sizeof(e->prev_torque));
  if (obs) get_obs(m, e, obs);
  memcpy(e->prev_prediction, action, nu * sizeof(double));
  /* domain randomisation after the observation (base_humanoid_env.py:228-233); decisions on stream 0 lanes 2, 3 */
  if (m->dynrand_interval > 0 || m->perturb_interval > 0) {
    uint32_t w[4];
    orc_philox(e->seed, e->env_id, e->rng_ctr, 0, w);
    if (m->dynrand_interval > 0 && randint(w[2], m->dynrand_interval) == 0) randomize_dynamics(m, e);
    if (m->perturb_interval > 0 && randint(w[3], m->perturb_interval) == 0) apply_perturbation(m, e);
  }
  double sum = 0;
  for (int i = 0; i < ORC_NREW; i++) sum += t[i];
  if (rew_terms) memcpy(rew_terms, t, sizeof(t));
  if (reward) *reward = sum;
  if (done) *done = d;
}

static void delay_orc_step_autoreset(const orc_model* m, orc_env* e, const double* action, int delay, int max_traj_len,
                                     double* obs, double* term_obs, double* rew_terms, double* reward, int* done, int* ended) {
  double r; int d;
  double o[ORC_NOBS];
  delay_orc_step(m, e, action, delay, o, rew_terms, &r, &d);
  e->traj_len++; e->ep_len++; e->ep_rew += r;
  int end = d || (e->traj_len >= max_traj_len);
  if (term_obs) memcpy(term_obs, o, m->nobs * sizeof(double));
  if (end) {
    e->status = 0;
    orc_reset(m, e, o);
  }
  if (obs) memcpy(obs, o, m->nobs * sizeof(double));
  if (reward) *reward = r;
  if (done) *done = d;
  if (ended) *ended = end;
}

/* one delayed control step with the RolloutWorker's auto-reset (orc_batch_step_autoreset's arguments + delay [n]), serially */
__attribute__((visibility("default"))) void delay_oracle_step(const orc_model* m, orc_env* envs, int n, const double* actions,
                                                                const int* delay, int max_traj_len, double* obs, double* term_obs,
                                                                double* rew_terms, double* reward, int* done, int* ended) {
  for (int i = 0; i < n; i++)
    delay_orc_step_autoreset(m, envs + i, actions + (size_t)i * m->nu, delay[i], max_traj_len, obs + (size_t)i * m->nobs,
                             term_obs + (size_t)i * m->nobs, rew_terms + (size_t)i * ORC_NREW, reward + i, done + i, ended + i);
}
