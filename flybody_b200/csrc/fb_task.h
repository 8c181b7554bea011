// fb_task.h -- device-side task logic (fb_task_program / fb_task_step): the reference's task hooks around the physics step, run by
// the task launches of fb_task_step (none of the seven step kernels calls it).
#pragma once
#include "fb_constraint.h"
//   ktask_reset  : composer auto-reset of envs whose last step was LAST -> initialize_episode (walk_imitation.py:112-136,
//                  flight_imitation.py:113-144): template state, root / ghost on the first reference row, wings on the beat
//                  pattern at a random phase (flight), optional U(-a, a) noise on listed joints; the env is held (not
//                  integrated) through the coming step, exactly as fb_reset_hold does for the host-side task code; with a
//                  dataset (ref_bank): the env's own reference cut from the trajectory bank first (ktask_reset_ref), walking:
//                  then the full-body start pose of the snippet and the wings back at their springs (ktask_reset3, ktask_reset4)
//   ktask_before : before_step (walk_imitation.py:138-150, flight_imitation.py:146-168): ghost root pose / velocity from
//                  the reference row of the current step; flight: one step of the wing-beat pattern generator at the requested
//                  frequency, wing force commands += pattern angle - wing angle (pattern_generators.py:131-203)
//   ktask_after  : check_termination, get_reward, get_discount (base.py:203-225, walk_imitation.py:179-203,
//                  flight_imitation.py:170-226) -> out[e] = reward, discount, step_type; walking with a dataset: the DeepMimic
//                  reward, its joint / site sums spread over the lanes first (ktask_reward)
// Scalar work runs on lane 0 (table scans of <= ~500 entries a few times per episode), array copies over the lanes.
FB_DEV unsigned tk_mix(unsigned x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }
FB_DEV float tk_u01(const DevTask& t, int e, int episode, int k) {
  return (float)(tk_mix(t.seed ^ tk_mix((unsigned)e * 0x9e3779b9u + (unsigned)episode * 0x85ebca6bu + (unsigned)k * 0xc2b2ae35u)) >> 8) * (1.0f / 16777216.0f);
}
// Model-parameter draws of a resetting env (fb_param_draws), the same device functions for fb_reset / fb_reset_hold and the device
// task's resets.  u is a counter hash of (seed, env, the env's draw count, parameter, element) in an index space of its own (an extra
// seed word); every lane reads the draw count, which kprm_count advances in a later phase.
FB_DEV float prm_u01(unsigned seed, int e, unsigned count, int p, int i) {
  return (float)(tk_mix(seed ^ 0x5bd1e995u ^ tk_mix((unsigned)e * 0x9e3779b9u + count * 0x85ebca6bu + ((unsigned)p << 24 | (unsigned)i) * 0xc2b2ae35u)) >> 8) *
         (1.0f / 16777216.0f);
}
FB_DEV void kprm_draw(const DevModel& m, const DevData& d, int e, int y) {
  if (!d.prm_draw) return;
  const DevPrmDraw& g = *d.prm_draw;
  const unsigned count = d.prm_count[e];
  float* row = d.prm + (size_t)e * d.prm_stride;
  for (int p = 0; p < FB_NPARAMS; p++) {
    if (!g.on[p]) continue;
    for (int i = y; i < g.n[p]; i += FB_NY) {
      const int s = d.prm_off[p] + (p == FB_P_BODY_INERTIA ? i + i / 3 : i);      // (body_inertia: four slots per body)
      const float lo = g.lo[s], hi = g.hi[s], u = prm_u01(g.seed, e, count, p, g.shared[p] ? 0 : i);
      row[s] = fminf(fmaxf(lo + u * (hi - lo), lo), hi);
      if (p == FB_P_DOF_DAMPING) row[d.prm_mdamp + m.dof_Madr[i]] = row[s];      // the diagonal of the implicit damping
    }
  }
}
FB_DEV void kprm_count(const DevData& d, int e, int y) { if (d.prm_draw && y == 0) d.prm_count[e]++; }
FB_DEV int wb_nearest(const DevTask& t, float f) {          // np.abs(beat_freqs - f).argmin(): first minimum
  int best = 0; float bd = fabsf(t.wb_freqs[0] - f);
  for (int i = 1; i < t.n_freq; i++) { float dd = fabsf(t.wb_freqs[i] - f); if (dd < bd) { bd = dd; best = i; } }
  return best;
}
FB_DEV int wb_argmin_phase(const float* tab, int n, float target) {
  int best = 0; float bd = fabsf(target - tab[0]);
  for (int i = 1; i < n; i++) { float dd = fabsf(target - tab[i]); if (dd < bd) { bd = dd; best = i; } }
  return best;
}
// the counters of an episode that starts in this step: time, flags, held through the step (as fb_reset_hold holds it), step 0.
// has_uniform is left to the caller: the other lanes of ktask_reset_vision still read it, and ktask_commit clears it there.
FB_DEV void tk_episode_start(const DevData& d, const DevTask& t, int e) {
  AT(d.time, 0) = 0; AT(d.flags, 0) = 0; AT(d.hold, 0) = 1; AT(d.prev_n, 0) = 0;
  t.step[e] = 0;
}
// FB_TASK_VISION (vision_guided_flight).  Height of a heightfield at the grid point nearest to (x, y): VisionFlightImitationWBPG.get_hfield_height
// (tasks/vision_flight.py:81-95: argmin of |axis - x| over linspace(-half, half, n); first minimum on ties)
FB_DEV float tk_hf_nearest(const DevTask& t, const float* h, float x, float y) {
  const float step = 2.0f * t.hf_half / (float)(t.hf_ncol - 1);
  int xi = (int)ceilf((x + t.hf_half) / step - 0.5f), yi = (int)ceilf((y + t.hf_half) / step - 0.5f);
  xi = xi < 0 ? 0 : (xi > t.hf_ncol - 1 ? t.hf_ncol - 1 : xi); yi = yi < 0 ? 0 : (yi > t.hf_nrow - 1 ? t.hf_nrow - 1 : yi);
  return h[(size_t)yi * t.hf_ncol + xi];
}
FB_DEV float tk_draw(const DevTask& t, int e, int episode, int k) { return t.has_uniform[e] ? t.uniform[8 * e + k] : tk_u01(t, e, episode, 16 + k); }
// terrain `pick` of the bank into the env's heightfield, block maxima and highest point (all lanes): a reset's, and a loaded state row's
FB_DEV void tk_terrain_copy(const DevTask& t, int e, int y, int pick) {
  const size_t cells = (size_t)t.hf_nrow * t.hf_ncol;
  const float* src = t.bank + cells * pick;
  float* dst = t.hf_data + cells * e;
  for (size_t i = y; i < cells; i += FB_NY) dst[i] = src[i];
  for (int i = y; i < t.hf_ncm; i += FB_NY) t.hf_cmax[(size_t)t.hf_ncm * e + i] = t.bank_cmax[(size_t)t.hf_ncm * pick + i];
  if (y == 0) t.hf_hmax[e] = t.bank_hmax[pick];
}
// initialize_episode_mjcf + initialize_episode of the vision task (vision_flight.py:97-139): targets, start point, wing-beat phase, a
// terrain of the bank copied into the env's heightfield (all lanes), the fly in its hover pose `target_height` above the terrain at the
// target speed.  Draw order: target height, target speed, x, y, wing-beat phase, terrain.
FB_DEV void ktask_reset_vision(const DevModel& m, const DevData& d, const DevTask& t, int e, int y, int episode) {
  int pick = (int)(tk_draw(t, e, episode, 5) * (float)t.n_bank); pick = pick < 0 ? 0 : (pick >= t.n_bank ? t.n_bank - 1 : pick);
  const float* src = t.bank + (size_t)t.hf_nrow * t.hf_ncol * pick;
  tk_terrain_copy(t, e, y, pick);
  if (y != 0) return;
  t.pick[e] = pick;
  const float th = t.th_rng[0] + (t.th_rng[1] - t.th_rng[0]) * tk_draw(t, e, episode, 0), ts = t.ts_rng[0] + (t.ts_rng[1] - t.ts_rng[0]) * tk_draw(t, e, episode, 1);
  const float x = t.x_rng[0] + (t.x_rng[1] - t.x_rng[0]) * tk_draw(t, e, episode, 2), yy = t.y_rng[0] + (t.y_rng[1] - t.y_rng[0]) * tk_draw(t, e, episode, 3);
  t.target[2 * e] = th; t.target[2 * e + 1] = ts;
  AT(d.qpos, t.root_qadr) = x; AT(d.qpos, t.root_qadr + 1) = yy; AT(d.qpos, t.root_qadr + 2) = tk_hf_nearest(t, src, x, yy) + th;
  for (int i = 0; i < 4; i++) AT(d.qpos, t.root_qadr + 3 + i) = t.hover_quat[i];
  const float phase = tk_draw(t, e, episode, 4);
  const int idx = wb_nearest(t, t.wb_base_freq);
  int pos = wb_argmin_phase(t.wb_phase + (size_t)idx * t.tab_len, t.tab_len, phase);
  const float* q0 = t.wb_traj + ((size_t)idx * t.tab_len + pos) * t.n_wing;
  for (int i = 0; i < t.n_wing; i++) AT(d.qpos, t.wing_qadr[i]) = q0[i];        // (the vision task starts the wings at rest: vision_flight.py:131-134)
  AT(d.qvel, t.root_vadr) = ts;
  t.wb_freq[e] = t.wb_base_freq; t.wb_idx[e] = idx; t.wb_pos[e] = pos;
  tk_episode_start(d, t, e);          // (has_uniform is read by every lane above: ktask_commit clears it)
}
// ref_bank (flight_imitation with a dataset, flight_imitation.py:88-111, trajectory_loaders.py:109-121; walk_imitation with a dataset,
// walk_imitation.py:93-110, trajectory_loaders.py:146-156, start always 0): the episode's trajectory and start step -- the pin of
// fb_task_ref_pick, else the counter hash (draw indices 256, 257: past the wing-beat phase's 0 and the noise joints' 1 + i).  Every lane
// computes the same pick.
FB_DEV void tk_ref_pick(const DevTask& t, int e, int episode, int& traj, int& start) {
  const int* pin = t.pin + 3 * (size_t)e;
  if (pin[0]) { traj = pin[1]; start = pin[2]; return; }
  int k = (int)floorf(tk_u01(t, e, episode, 256) * (float)t.n_pick); k = k > t.n_pick - 1 ? t.n_pick - 1 : k;
  traj = t.pick_traj[k];
  const int span = t.traj_len[traj] - t.start_margin;
  start = 0;
  if (t.randomize_start) { start = (int)floorf(tk_u01(t, e, episode, 257) * (float)span); start = start > span - 1 ? span - 1 : start; }
}
// the env's reference of the new episode: rows start .. start + n of its trajectory into its slot, root x, y relative to the x, y in
// columns 13, 14 of row `start` (flight: the CoM's, walking: the root's), the rest of the slot padded with the last row (as the host-side
// code fills a slot); root and ghost on row `start`, read from the bank because the other lanes are still writing the slot
FB_DEV void ktask_reset_ref(const DevModel& m, const DevData& d, const DevTask& t, int e, int y, int episode) {
  int traj, start; tk_ref_pick(t, e, episode, traj, start);
  const int len = t.traj_len[traj], row0 = t.traj_off[traj] + start;
  const int n = len - start < t.slot_len ? len - start : t.slot_len;
  const float* b0 = t.rbank + (size_t)t.rbank_w * row0;
  const float cx = b0[13], cy = b0[14];
  float* slot = t.slots + (size_t)e * 7 * t.slot_len;
  for (int i = y; i < t.slot_len; i += FB_NY) {
    const float* r = t.rbank + (size_t)t.rbank_w * (row0 + (i < n ? i : n - 1));
    float* o = slot + 7 * (size_t)i;
    o[0] = r[0] - cx; o[1] = r[1] - cy;
    for (int c = 2; c < 7; c++) o[c] = r[c];
  }
  if (y < 7) {
    const float r = y == 0 ? b0[0] - cx : (y == 1 ? b0[1] - cy : b0[y]);
    AT(d.qpos, t.root_qadr + y) = r;
    if (t.ghost_qadr >= 0) AT(d.qpos, t.ghost_qadr + y) = r + (y < 3 ? t.ghost_offset[y] : 0.0f);
  }
  if (y == 0) {
    if (t.kind == FB_TASK_FLIGHT) for (int i = 0; i < 3; i++) AT(d.qvel, t.root_vadr + i) = b0[7 + i];      // (walking starts at rest)
    const int rows = n < t.max_episode_rows ? n : t.max_episode_rows;
    t.ep_traj[e] = traj; t.ep_start[e] = start; t.ep_row0[e] = row0; t.ep_n[e] = n; t.ep_steps[e] = rows - (t.future_steps + 1);
  }
}
FB_DEV void ktask_reset(const DevModel& m, const DevData& d, int e, int y) {
  if (!d.task || e >= d.N) return;
  const DevTask& t = *d.task;
  if (!t.needs_reset[e]) return;
  for (int i = y; i < m.nq; i += FB_NY) AT(d.qpos, i) = t.reset_qpos[i];
  for (int i = y; i < m.nv; i += FB_NY) { AT(d.qvel, i) = 0.0f; AT(d.qacc, i) = 0.0f; }
  for (int i = y; i < m.na; i += FB_NY) AT(d.act, i) = 0.0f;
  for (int i = y; i < m.nu; i += FB_NY) AT(d.ctrl, i) = 0.0f;      // physics.reset() = mj_resetData: the FIRST observation does not see the old controls
  zero_applied(m, d, e, y);
  kprm_draw(m, d, e, y);
}
FB_DEV void ktask_reset2(const DevModel& m, const DevData& d, int e, int y) {      // after the template copy (other lanes wrote it)
  if (!d.task || e >= d.N) return;
  const DevTask& t = *d.task;
  if (!t.needs_reset[e]) return;
  kprm_count(d, e, y);                     // (every lane read the draw count in ktask_reset)
  const int episode = t.episode[e];
  if (t.kind == FB_TASK_VISION) { ktask_reset_vision(m, d, t, e, y, episode); return; }
  if (t.kind == FB_TASK_TEMPLATE || t.kind == FB_TASK_BALL) {          // the template pose as copied, at rest (no reference, no ghost)
    if (y == 0) { tk_episode_start(d, t, e); t.has_uniform[e] = 0; }
    return;
  }
  if (t.ref_bank) ktask_reset_ref(m, d, t, e, y, episode);
  else if (y < 7) { float r = t.ref_qpos[y]; AT(d.qpos, t.root_qadr + y) = r; if (t.ghost_qadr >= 0) AT(d.qpos, t.ghost_qadr + y) = r + (y < 3 ? t.ghost_offset[y] : 0.0f); }
  if (y == 0) {
    if (t.kind == FB_TASK_FLIGHT) {          // wings on the beat pattern of the base frequency at a random phase, root at the reference speed
      float phase = t.has_uniform[e] ? t.uniform[8 * e] : tk_u01(t, e, episode, 0);
      int idx = wb_nearest(t, t.wb_base_freq), len = t.wb_len[idx];
      int pos = wb_argmin_phase(t.wb_phase + (size_t)idx * t.tab_len, t.tab_len, phase);
      int nxt = pos + 1 < len ? pos + 1 : len - 1;
      const float* q0 = t.wb_traj + ((size_t)idx * t.tab_len + pos) * t.n_wing; const float* q1 = t.wb_traj + ((size_t)idx * t.tab_len + nxt) * t.n_wing;
      for (int i = 0; i < t.n_wing; i++) { AT(d.qpos, t.wing_qadr[i]) = q0[i]; AT(d.qvel, t.wing_vadr[i]) = (q1[i] - q0[i]) / t.dt; }
      if (!t.ref_bank) for (int i = 0; i < 3; i++) AT(d.qvel, t.root_vadr + i) = t.ref_qvel[i];
      t.wb_freq[e] = t.wb_base_freq; t.wb_idx[e] = idx; t.wb_pos[e] = pos;
    }
    tk_episode_start(d, t, e);
    t.has_uniform[e] = 0;          // (the episode counter, read by every lane above, advances in ktask_before)
  }
}
// The later writes of a reset each take a phase of their own, after the write they build on: the dataset's joint list may include the
// wings, and the noise joints are among its joints, so different lanes write and add to the same qpos entries (walk_imitation.py:112-136).
// walking with a dataset: the mocap joints at row `start` of the snippet (the full-body start pose, walk_imitation.py:117-118)
FB_DEV void ktask_reset3(const DevModel& m, const DevData& d, int e, int y) {
  if (!d.task || e >= d.N) return;
  const DevTask& t = *d.task;
  if (t.kind != FB_TASK_WALK || !t.ref_bank || !t.needs_reset[e]) return;
  const float* b0 = t.rbank + (size_t)t.rbank_w * t.ep_row0[e] + 15;
  for (int i = y; i < t.n_mjnt; i += FB_NY) AT(d.qpos, t.mocap_qadr[i]) = b0[i];
}
// ... then the wings back at their spring references (walk_imitation.py:119-121)
FB_DEV void ktask_reset4(const DevModel& m, const DevData& d, int e, int y) {
  if (!d.task || e >= d.N) return;
  const DevTask& t = *d.task;
  if (t.kind != FB_TASK_WALK || !t.ref_bank || !t.needs_reset[e]) return;
  for (int i = y; i < t.n_wing; i += FB_NY) AT(d.qpos, t.wing_qadr[i]) = t.wing_spring[i];
}
// ... then the optional U(-a, a) noise on the listed joints
FB_DEV void ktask_reset5(const DevModel& m, const DevData& d, int e, int y) {
  if (!d.task || e >= d.N) return;
  const DevTask& t = *d.task;
  if (t.kind == FB_TASK_VISION || !t.needs_reset[e]) return;
  const int episode = t.episode[e];
  for (int i = y; i < t.n_noise; i += FB_NY) AT(d.qpos, t.noise_qadr[i]) += t.noise_amp * (2.0f * tk_u01(t, e, episode, 1 + i) - 1.0f);
}
FB_DEV void ktask_before(const DevModel& m, const DevData& d, int e, int y) {
  if (!d.task || e >= d.N) return;
  const DevTask& t = *d.task;
  const int resetting = t.needs_reset[e];
  int step = resetting ? 0 : t.step[e];
  // the shared reference, or (ref_bank) the env's own: pose from its slot, velocity from the bank, step clamped by its rows in use
  const int last = t.ref_bank ? t.ep_n[e] - 1 : t.ref_len - 1;
  if (step > last) step = last;
  if (t.ghost_qadr >= 0) {
    const float* rq = t.ref_bank ? t.slots + ((size_t)e * t.slot_len + step) * 7 : t.ref_qpos + 7 * step;
    const float* rv = t.ref_bank ? t.rbank + (size_t)t.rbank_w * (t.ep_row0[e] + step) + 7 : t.ref_qvel + 6 * step;
    if (y < 7) AT(d.qpos, t.ghost_qadr + y) = rq[y] + (y < 3 ? t.ghost_offset[y] : 0.0f);
    else if (y < 13) AT(d.qvel, t.ghost_vadr + y - 7) = resetting ? 0.0f : rv[y - 7];
  }
  if (y == 0) {
    if ((t.kind == FB_TASK_FLIGHT || t.kind == FB_TASK_VISION) && !resetting) {
      float a = t.user_col >= 0 ? d.sc_vals[(size_t)e * d.sc_k + t.user_col] : 0.0f;
      if (!(a == a)) a = 0.0f;
      float ctrl_freq = t.wb_base_freq * (1.0f + t.wb_rel_range * a);
      int idx = t.wb_idx[e], pos = (t.wb_pos[e] + 1) % t.wb_len[idx];
      float f = t.wb_rate != 0.0f ? t.wb_freq[e] * t.wb_rate + ctrl_freq * (1.0f - t.wb_rate) : ctrl_freq;
      int nw = wb_nearest(t, f);
      if (nw != idx) {          // keep the phase within the beat when changing table
        float cur = t.wb_phase_mod[(size_t)idx * t.tab_len + pos];
        pos = wb_argmin_phase(t.wb_phase_mod + (size_t)nw * t.tab_len, t.tab_len, cur);
        idx = nw;
      }
      t.wb_freq[e] = f; t.wb_idx[e] = idx; t.wb_pos[e] = pos;
      const float* tg = t.wb_traj + ((size_t)idx * t.tab_len + pos) * t.n_wing;
      for (int i = 0; i < t.n_wing; i++) AT(d.ctrl, t.wing_ctrl[i]) += tg[i] - AT(d.qpos, t.wing_qadr[i]);
    }
  }
}
// counters advance in a phase of their own: every lane of ktask_before reads the step it is about to leave
FB_DEV void ktask_commit(const DevModel& m, const DevData& d, int e, int y) {
  if (!d.task || e >= d.N || y != 0) return;
  const DevTask& t = *d.task;
  const int resetting = t.needs_reset[e];
  t.resetting[e] = resetting;
  if (resetting) { t.episode[e] = t.episode[e] + 1; t.has_uniform[e] = 0; if (t.ref_bank) t.pin[3 * (size_t)e] = 0; } else t.step[e] = t.step[e] + 1;
  t.op_step[e] = t.step[e]; t.op_first[e] = (unsigned char)resetting;
}
FB_DEV float tk_lin_tol(float x, float margin) { float v = 1.0f - fabsf(x) / margin; return v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v); }
// quaternions.py:215-333 restated in fp32: quat_z2vec with its exact-zero edge cases (vec = (0, 0, z): identity, or the half turn about x
// for z < 0), axis_angle_to_quat, joint_orientation_quat and the short-arc distance acos(min(1, 2 (p.q)^2 - 1)) of normalised quaternions
FB_DEV Q4 tk_quat_z2vec(V3 v) {
  if (v.x == 0.0f && v.y == 0.0f) return v.z < 0.0f ? q4(0.0f, 1.0f, 0.0f, 0.0f) : q4(1.0f, 0.0f, 0.0f, 0.0f);
  const float n = sqrtf(v.x * v.x + v.y * v.y + v.z * v.z);
  const float ux = v.x / n, uy = v.y / n, uz = v.z / n, an = sqrtf(uy * uy + ux * ux);
  const float h = 0.5f * acosf(uz > 1.0f ? 1.0f : (uz < -1.0f ? -1.0f : uz)), s = sinf(h);      // (|uz| > 1 only by rounding)
  return q4(cosf(h), s * (-uy / an), s * (ux / an), 0.0f);
}
FB_DEV Q4 tk_axis_angle_quat(V3 a, float angle) {
  const float n = sqrtf(a.x * a.x + a.y * a.y + a.z * a.z), h = 0.5f * angle, s = sinf(h);
  return q4(cosf(h), s * (a.x / n), s * (a.y / n), s * (a.z / n));
}
FB_DEV Q4 tk_joint_quat(V3 axis, float qpos) { return qmul(tk_axis_angle_quat(axis, qpos), tk_quat_z2vec(axis)); }
FB_DEV float tk_quat_dist(Q4 p, Q4 q) {
  const float np_ = sqrtf(p.w * p.w + p.x * p.x + p.y * p.y + p.z * p.z), nq = sqrtf(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
  const float c = (p.w / np_) * (q.w / nq) + (p.x / np_) * (q.x / nq) + (p.y / np_) * (q.y / nq) + (p.z / np_) * (q.z / nq);
  const float x = 2.0f * c * c - 1.0f;
  return acosf(x < 1.0f ? x : 1.0f);
}
// walking with a dataset: the bank row of the reference features at the env's step (rewards.py:66-83: the row of step min(step, n - 1))
FB_DEV const float* tk_walk_ref_row(const DevTask& t, int e) {
  const int s = t.step[e], last = t.ep_n[e] - 1;
  return t.rbank + (size_t)t.rbank_w * (t.ep_row0[e] + (s < last ? s : last));
}
// ... the DeepMimic terms over the dataset's joints and sites, lanes over joints / sites (rewards.py:10-63): squared mocap qvel errors,
// squared end-effector (root2site) errors, squared short-arc angles between the joint orientations; per-lane sums to rw_part
FB_DEV void ktask_reward(const DevModel& m, const DevData& d, int e, int y) {
  if (!d.task || !d.tobs || e >= d.N) return;
  const DevTask& t = *d.task;
  if (t.kind != FB_TASK_WALK || !t.ref_bank) return;
  const float* o = d.tobs + (size_t)e * d.tobs_dim;
  const int nj = t.n_mjnt, ns = t.n_msite;
  const float* rqv = tk_walk_ref_row(t, e) + 15 + nj;
  const float* rsite = rqv + nj;
  const float* rjq = rsite + 3 * ns;
  float sv = 0.0f, ss = 0.0f, sq = 0.0f;
  for (int i = y; i < nj; i += FB_NY) {
    const float dv = o[t.obs_mocap_qvel_off + i] - rqv[i];
    sv += dv * dv;
    const float* a = o + t.obs_mocap_axes_off + 3 * i;
    const float ang = tk_quat_dist(tk_joint_quat(v3(a[0], a[1], a[2]), o[t.obs_mocap_qpos_off + i]), q4(rjq[4 * i], rjq[4 * i + 1], rjq[4 * i + 2], rjq[4 * i + 3]));
    sq += ang * ang;
  }
  for (int i = y; i < 3 * ns; i += FB_NY) { const float ds = o[t.obs_mocap_sites_off + i] - rsite[i]; ss += ds * ds; }
  float* p = t.rw_part + ((size_t)e * FB_NY + y) * 3;
  p[0] = sv; p[1] = ss; p[2] = sq;
}
// ... and on lane 0: the root terms, the lanes' sums in lane order, the product of the four DeepMimic factors (weights 20, 1, 1, 1) and the
// six wing-retraction factors (walk_imitation.py:152-177).  The CoM feature is the snippet's root position shifted as the loader shifts it.
FB_DEV float tk_walk_reward(const DevTask& t, int e, const float* o) {
  const float* r = tk_walk_ref_row(t, e);
  const float* b0 = t.rbank + (size_t)t.rbank_w * t.ep_row0[e];
  const float* rp = o + t.obs_root_pose_off;
  const float* rv = o + t.obs_root_qvel_off;
  const float c0 = rp[0] - (r[0] - b0[13]), c1 = rp[1] - (r[1] - b0[14]), c2 = rp[2] - r[2];
  const float d_com = c0 * c0 + c1 * c1 + c2 * c2;
  float d_qvel = 0.0f, d_site = 0.0f;
  for (int k = 0; k < 6; k++) { const float dv = rv[k] - r[7 + k]; d_qvel += dv * dv; }
  const float a = tk_quat_dist(q4(rp[3], rp[4], rp[5], rp[6]), q4(r[3], r[4], r[5], r[6]));
  float d_quat = a * a;
  for (int l = 0; l < FB_NY; l++) { const float* p = t.rw_part + ((size_t)e * FB_NY + l) * 3; d_qvel += p[0]; d_site += p[1]; d_quat += p[2]; }
  auto factor = [&](int k, float diff) { return expf(-0.5f / (t.dm_std[k] * t.dm_std[k]) * diff) * t.dm_weight[k]; };
  float reward = factor(0, d_com) * factor(1, d_qvel) * factor(2, d_site) * factor(3, d_quat);
  for (int i = 0; i < t.n_wing; i++) reward *= tk_lin_tol(o[t.obs_wing_qpos_off + i] - t.wing_spring[i], t.retract_margin);
  return reward;
}
// |velocimeter| and |gyro| at the last substep: the walker's speed terminations (walk_imitation.py:179-203, walk_on_ball.py:75-81)
FB_DEV void tk_walker_speeds(const DevData& d, const DevTask& t, int e, float& linvel, float& angvel) {
  const float* lv = &AT(d.sensordata, t.velocimeter_adr); const float* av = &AT(d.sensordata, t.gyro_adr);
  linvel = sqrtf(lv[0] * lv[0] + lv[1] * lv[1] + lv[2] * lv[2]); angvel = sqrtf(av[0] * av[0] + av[1] * av[1] + av[2] * av[2]);
}
// get_discount and the step type (base.py:203-225): out[e] = reward, discount, step_type (0 FIRST, 1 MID, 2 LAST), 0.  An env that started
// its episode in this step reports FIRST, reward 0, discount 1; a termination costs the discount unless end_ok (walk / flight: end of reference)
FB_DEV void tk_end_step(const DevTask& t, int e, bool resetting, bool terminate, bool end_ok, float reward, int step_now) {
  const bool last = terminate || (double)step_now * (double)t.dt >= (double)t.time_limit - 1e-9;
  float* out = t.out + 4 * (size_t)e;
  out[0] = resetting ? 0.0f : reward;
  out[1] = resetting ? 1.0f : ((terminate && !end_ok) ? 0.0f : 1.0f);
  out[2] = resetting ? 0.0f : (last ? 2.0f : 1.0f);
  out[3] = 0.0f;
  t.needs_reset[e] = (last && !resetting) ? 1 : 0;
}
FB_DEV void ktask_after(const DevModel& m, const DevData& d, int e, int y) {
  if (!d.task || !d.tobs || e >= d.N || y != 0) return;
  const DevTask& t = *d.task;
  const float* o = d.tobs + (size_t)e * d.tobs_dim;
  const int resetting = t.resetting[e], step_now = t.step[e];
  const float* rd = o + t.obs_refdisp_off;
  const float com_dist = sqrtf(rd[0] * rd[0] + rd[1] * rd[1] + rd[2] * rd[2]);
  const bool reached_end = step_now == t.ep_steps[e];
  float s2 = 0; for (int i = 0; i < m.nv; i++) { float x = AT(d.qacc, i); s2 += x * x; }
  const bool bad = (AT(d.flags, 0) & 1) != 0 || !(sqrtf(s2) <= t.term_qacc);      // bits 1, 2 are capacity overflows, not bad physics
  bool terminate; float reward = 1.0f, linvel, angvel;
  if (t.kind == FB_TASK_TEMPLATE) {      // template_task (tasks/template_task.py): reward 1; only a bad state ends an episode early
    terminate = bad;
  } else if (t.kind == FB_TASK_BALL) {      // walk_on_ball (tasks/walk_on_ball.py:55-81): ball-velocity reward; velocimeter / gyro / bad state end an episode
    tk_walker_speeds(d, t, e, linvel, angvel);
    terminate = linvel > t.term_linvel || angvel > t.term_angvel || bad;
    for (int i = 0; i < 3; i++) reward *= tk_lin_tol(AT(d.qvel, t.ball_vadr + i) - t.ball_target[i], t.ball_margin);
  } else if (t.kind == FB_TASK_VISION) {      // vision_flight.py:157-254: reward factors, fatal contacts with world geoms
    const float th = t.target[2 * e], ts = t.target[2 * e + 1];
    const float x = AT(d.qpos, t.root_qadr), yy = AT(d.qpos, t.root_qadr + 1), z = AT(d.qpos, t.root_qadr + 2);
    const float vx = AT(d.qvel, t.root_vadr), vy = AT(d.qvel, t.root_vadr + 1), vz = AT(d.qvel, t.root_vadr + 2);
    auto lin = [](float v, float lo, float hi, float margin) { float dd = v < lo ? lo - v : (v > hi ? v - hi : 0.0f); dd /= margin; return dd <= 0.0f ? 1.0f : (dd >= 1.0f ? 0.0f : 1.0f - dd); };
    const float height = lin(z - tk_hf_nearest(t, t.hf_data + (size_t)t.hf_nrow * t.hf_ncol * e, x, yy), th, th, 0.15f);
    const float x_speed = lin(vx, ts, 3.0e38f, 1.1f * ts), speed = lin(sqrtf(vx * vx + vy * vy + vz * vz), ts, ts, 1.1f * ts);
    const float side = lin(AT(d.sensordata, t.velocimeter_adr + 1), 0.0f, 0.0f, 10.0f);
    const M3 R = ld9(d.xmat, t.root_body, d, e);
    float c = R.m[6] * t.target_zaxis[0] + R.m[7] * t.target_zaxis[1] + R.m[8] * t.target_zaxis[2]; c = c < -1.0f ? -1.0f : (c > 1.0f ? 1.0f : c);
    const float zax = lin(acosf(c), 0.0f, 0.0f, 3.14159265358979f);
    float centre = 1.0f;      // 'trench' arenas: distance to the corridor's centre line at the nearest of its sample points (the lower one on ties)
    if (t.trench_cap > 0) {
      const int pk = t.pick[e], tn = t.trench_len[pk]; const float x0 = t.trench_x[2 * pk], x1 = t.trench_x[2 * pk + 1];
      if (x >= x0 && x <= x1) {
        const float u = (x - x0) / (x1 - x0) * (float)(tn - 1);
        int idx = (int)floorf(u); if (u - (float)idx > 0.5f) idx++;
        idx = idx < 0 ? 0 : (idx > tn - 1 ? tn - 1 : idx);
        const float yc = t.trench_y[(size_t)pk * t.trench_cap + idx];
        centre = lin(yy, yc, yc, 0.15f);
      }
    }
    reward = height * x_speed * speed * side * zax * centre;
    bool contact = false;
    if (t.fatal) { const int nc = AT(d.ncon, 0); for (int ci = 0; ci < nc; ci++) if (AT(d.con_efcadr, ci) >= 0 && (m.geom_bodyid[AT(d.con_geom1, ci)] == 0 || m.geom_bodyid[AT(d.con_geom2, ci)] == 0)) contact = true; }
    terminate = bad || contact;
  } else if (t.kind == FB_TASK_WALK) {
    tk_walker_speeds(d, t, e, linvel, angvel);
    terminate = linvel > t.term_linvel || angvel > t.term_angvel || reached_end || com_dist > t.term_com || bad;
    reward = t.ref_bank ? tk_walk_reward(t, e, o) : 1.0f;      // inference mode: reward factors == (1,)
  } else {
    const float height = AT(d.qpos, t.root_qadr + 2);
    terminate = height < t.term_height || com_dist > t.term_com || reached_end || bad;
    // reward: CoM displacement and orientation error to the ghost (flight_imitation.py:190-212; legs disabled: third factor 1)
    V3 gp = v3(AT(d.qpos, t.ghost_qadr), AT(d.qpos, t.ghost_qadr + 1), AT(d.qpos, t.ghost_qadr + 2));      // the ghost as placed (offset included)
    Q4 gq = q4(AT(d.qpos, t.ghost_qadr + 3), AT(d.qpos, t.ghost_qadr + 4), AT(d.qpos, t.ghost_qadr + 5), AT(d.qpos, t.ghost_qadr + 6));
    V3 gcom = gp + mul(q2m(gq), v3(t.com_offset[0], t.com_offset[1], t.com_offset[2]));
    float mass = AT(d.crb10, FB_I10S * t.com_body);
    V3 com = v3(AT(d.crb10, FB_I10S * t.com_body + 1), AT(d.crb10, FB_I10S * t.com_body + 2), AT(d.crb10, FB_I10S * t.com_body + 3)) * (mass > 0 ? 1.0f / mass : 0.0f)
             + v3(AT(d.ref, 0), AT(d.ref, 1), AT(d.ref, 2));
    V3 dv = gcom - com; float disp = sqrtf(dot(dv, dv));
    const float* rq = o + t.obs_refquat_off;
    float n2 = rq[0] * rq[0] + rq[1] * rq[1] + rq[2] * rq[2] + rq[3] * rq[3];
    float x = 2.0f * (rq[0] * rq[0] / n2) - 1.0f; if (x > 1.0f) x = 1.0f;
    reward = tk_lin_tol(disp, 0.4f) * tk_lin_tol(acosf(x), 3.14159265358979f);
  }
  const bool imitation = t.kind == FB_TASK_WALK || t.kind == FB_TASK_FLIGHT;
  tk_end_step(t, e, resetting, terminate, imitation && reached_end, reward, step_now);
}
