/* flybody_b200.h -- C ABI of the H100-native batched fruit-fly physics stepper.
 *
 * The reference (TuragaLab/flybody) has no FFI of its own: the hot path sits behind
 * dm_control's `Physics.step()` which `composer.Environment.step()` calls n_sub_steps times per
 * control step (reference flybody/fly_envs.py:152-155; SURVEY.md 3.3 / 8(b)).  These entry
 * points are what a ctypes binding replacing that `physics.step()` loop binds to; each one
 * names the reference-side call it stands in for.
 *
 * Conventions: plain C, no torch types.  Return 0 on success, negative code on error
 * (message via fb_last_error).  Caller owns host buffers; the library owns device buffers.
 * One handle = one device + one stream; calls on a handle are not re-entrant.
 * Device side: one fp32/int32 record per env (one warp steps one env); host-side buffers passed to fb_*
 * are rows [env][component] (what numpy/dm_env code holds).
 *
 * flybody_b200/abi.py binds this header from its text: prototypes, enums (with explicit values), integer #defines and
 * structs of scalar, pointer and array fields.  It refuses any other construct or type, naming the line.
 */
#ifndef FLYBODY_B200_H_
#define FLYBODY_B200_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* enums shared by compiler (Python), oracle (C) and kernels (CUDA) */
enum { FB_GEOM_PLANE = 0, FB_GEOM_SPHERE = 2, FB_GEOM_CAPSULE = 3, FB_GEOM_ELLIPSOID = 4,
       FB_GEOM_CYLINDER = 5, FB_GEOM_BOX = 6 };
enum { FB_JNT_FREE = 0, FB_JNT_BALL = 1, FB_JNT_HINGE = 3 };
enum { FB_TRN_JOINT = 0, FB_TRN_TENDON = 1, FB_TRN_BODY = 2 };
enum { FB_DYN_NONE = 0, FB_DYN_FILTER = 2, FB_DYN_FILTEREXACT = 3 };
enum { FB_SENS_TOUCH = 0, FB_SENS_ACCELEROMETER = 1, FB_SENS_VELOCIMETER = 2, FB_SENS_GYRO = 3,
       FB_SENS_FORCE = 4 };

/* Flat model = the subset of mjModel the fly's mj_step touches (generated from
 * flybody_b200/flymodel.py:FIELDS; tests/test_model.py keeps the two in sync). */
/*@FBMODEL_BEGIN*/
typedef struct FbModel {
  int32_t nq;
  int32_t nv;
  int32_t nu;
  int32_t na;
  int32_t nbody;
  int32_t njnt;
  int32_t ngeom;
  int32_t npair;
  int32_t nsite;
  int32_t ntendon;
  int32_t nwrap;
  int32_t nsensor;
  int32_t nsensordata;
  int32_t nM;
  int32_t nfluid;
  int32_t opt_iterations;
  int32_t opt_ls_iterations;
  int32_t opt_noslip_iterations;
  int32_t opt_cone_elliptic;
  double opt_timestep;
  double opt_gravity[3];
  double opt_density;
  double opt_viscosity;
  double opt_wind[3];
  double opt_impratio;
  double opt_tolerance;
  double opt_ls_tolerance;
  double opt_noslip_tolerance;
  double stat_meaninertia;
  const int32_t* body_parentid;
  const int32_t* body_rootid;
  const int32_t* body_jntadr;
  const int32_t* body_jntnum;
  const int32_t* body_dofadr;
  const int32_t* body_dofnum;
  const int32_t* body_lastdof;
  const int32_t* body_fluid_ellipsoid;
  const double* body_pos;
  const double* body_quat;
  const double* body_ipos;
  const double* body_iquat;
  const double* body_mass;
  const double* body_inertia;
  const double* body_invweight0;
  const double* body_subtreemass;
  const int32_t* jnt_type;
  const int32_t* jnt_qposadr;
  const int32_t* jnt_dofadr;
  const int32_t* jnt_bodyid;
  const int32_t* jnt_limited;
  const double* jnt_pos;
  const double* jnt_axis;
  const double* jnt_stiffness;
  const double* jnt_range;
  const double* jnt_solref;
  const double* jnt_solimp;
  const double* jnt_margin;
  const double* qpos0;
  const double* qpos_spring;
  const int32_t* dof_bodyid;
  const int32_t* dof_jntid;
  const int32_t* dof_parentid;
  const int32_t* dof_Madr;
  const double* dof_armature;
  const double* dof_damping;
  const double* dof_invweight0;
  const int32_t* geom_type;
  const int32_t* geom_bodyid;
  const int32_t* geom_condim;
  const int32_t* geom_priority;
  const double* geom_size;
  const double* geom_pos;
  const double* geom_quat;
  const double* geom_rbound;
  const double* geom_friction;
  const double* geom_solmix;
  const double* geom_solref;
  const double* geom_solimp;
  const double* geom_margin;
  const double* geom_gap;
  const int32_t* pair_geom1;
  const int32_t* pair_geom2;
  const int32_t* fluid_bodyid;
  const double* fluid_pos;
  const double* fluid_quat;
  const double* fluid_size;
  const double* fluid_coef;
  const int32_t* site_bodyid;
  const int32_t* site_type;
  const double* site_pos;
  const double* site_quat;
  const double* site_size;
  const int32_t* tendon_adr;
  const int32_t* tendon_num;
  const int32_t* wrap_dofid;
  const int32_t* wrap_qposadr;
  const double* wrap_coef;
  const int32_t* actuator_trntype;
  const int32_t* actuator_trnid;
  const int32_t* actuator_dyntype;
  const int32_t* actuator_biastype;
  const int32_t* actuator_ctrllimited;
  const int32_t* actuator_forcelimited;
  const int32_t* actuator_actadr;
  const double* actuator_dynprm;
  const double* actuator_gainprm;
  const double* actuator_biasprm;
  const double* actuator_ctrlrange;
  const double* actuator_forcerange;
  const int32_t* sensor_type;
  const int32_t* sensor_objid;
  const int32_t* sensor_adr;
  const int32_t* sensor_dim;
} FbModel;
/*@FBMODEL_END*/

/* fields for fb_get / fb_set (per-env arrays; n = floats per env) */
enum FbField {
  FB_QPOS = 0,        /* nq   : physics.data.qpos                                   */
  FB_QVEL = 1,        /* nv   : physics.data.qvel                                   */
  FB_ACT = 2,         /* na   : physics.data.act                                    */
  FB_CTRL = 3,        /* nu   : physics.data.ctrl (physics.set_control)             */
  FB_QACC = 4,        /* nv   : physics.data.qacc (tasks/base.py:224)               */
  FB_QACC_WARMSTART = 5,
  FB_SENSORDATA = 6,  /* nsensordata : last-substep sensordata                      */
  FB_SENSOR_MEAN = 7, /* nsensordata : mean over the substeps of the last fb_step
                         (observable buffer_size + aggregator='mean', fruitfly.py:626-665) */
  FB_XPOS = 8,        /* nbody*3  : physics.bind(bodies).xpos                       */
  FB_XMAT = 9,        /* nbody*9  : physics.bind(bodies).xmat                       */
  FB_SITE_XPOS = 10,  /* nsite*3                                                    */
  FB_SITE_XMAT = 11,  /* nsite*9                                                    */
  FB_SUBTREE_COM = 12,/* nbody*3  : physics.data.subtree_com                        */
  FB_NCON = 13,       /* 1 (as float): number of detected contacts                  */
  FB_NEFC = 14,       /* 1 (as float): number of constraint rows                    */
  FB_TIME = 15,       /* 1 : physics.data.time                                      */
  FB_QFRC_SMOOTH = 16,/* nv : passive - bias + actuator                             */
  FB_QM_DENSE = 17,   /* nv*nv : dense joint-space inertia (debug / parity)         */
  FB_QFRC_CONSTRAINT = 18, /* nv                                                    */
  FB_SOLVER_NITER = 19,    /* 1                                                     */
  FB_QFRC_PASSIVE = 20,    /* nv                                                    */
  FB_QFRC_BIAS = 21,       /* nv                                                    */
  FB_QFRC_ACTUATOR = 22,   /* nv                                                    */
  FB_CONTACT = 23,    /* FB_MAXCON * 16: per contact [dist, pos3, normal3, geom1, geom2, dim, incl, mu, efc_adr, tangent3]
                         (tangent3: the frame's first tangent; the second is normal x tangent) */
  FB_EFC_FORCE = 24,  /* FB_MAXEFC                                                  */
  FB_FLAGS = 25,      /* 1 (as float): bit0 bad state (nan/inf or |qacc|>1e14), bit1 contact overflow, bit2 efc overflow */
  FB_QFRC_APPLIED = 26, /* nv : physics.data.qfrc_applied, generalized forces added to qfrc_smooth every substep           */
  FB_XFRC_APPLIED = 27, /* nbody*6 : physics.data.xfrc_applied, per body a world-frame force, then torque, applied at the
                           body's CoM (mj_xfrcAccumulate: qfrc_smooth += J^T wrench over the body's ancestor dofs).
                           Both (fb_set, fb_write_state, fb_get with is_device = 0) persist across substeps and steps until
                           overwritten, are zeroed for the envs of fb_reset / fb_reset_hold / a device-task reset
                           (mj_resetData), and read as zero while unset                                                  */
  FB_NFIELDS = 28
};

#define FB_MAXCON 64     /* contact slots per env   */
#define FB_MAXEFC 160    /* constraint rows per env */

typedef struct FbSim* FbHandle;

/* mjcf.Physics.from_mjcf_model + mj_makeData, batched: uploads the model, allocates SoA state
 * for n_envs environments on `device`, all envs at qpos0 / zero velocity.
 * Refuses (-3, fb_last_error says why) a model the step would integrate as something else: among others, a touch sensor on a site
 * that is neither a sphere nor a capsule (the touch ray test knows those two shapes only; MuJoCo ray-tests the site's own shape). */
int fb_create(const FbModel* m, int n_envs, int device, FbHandle* out);
int fb_destroy(FbHandle h);

/* physics.reset_context()/bind(...).qpos = ... (walk_imitation.py:112-136): overwrite qpos/qvel
 * of the listed envs (AoS host arrays [n][nq], [n][nv]; NULL = model defaults), zero act /
 * warm start / time, then mj_forward for those envs.  env_ids == NULL means all envs.        */
int fb_reset(FbHandle h, const int32_t* env_ids, int n, const float* qpos, const float* qvel);

/* Auto-reset of a subset of envs inside a batched rollout (composer.Environment resets an env on the step()
 * after a LAST timestep and returns the reset observation without stepping): writes the reset state of the
 * listed envs on the device and marks them "held" -- the next fb_step recomputes their forward quantities
 * every substep but does not integrate them; the hold is cleared when that fb_step completes.            */
int fb_reset_hold(FbHandle h, const int32_t* env_ids, int n, const float* qpos, const float* qvel);

/* physics.set_control(ctrl) (fruitfly.py:540-544).  ctrl: contiguous rows [N][nu], on the host
 * (is_device=0, copied asynchronously on the handle's stream) or already on the device (is_device=1). */
int fb_set_ctrl(FbHandle h, const float* ctrl, int is_device);
/* FruitFly.apply_action (fruitfly.py:532-544) on the device: after this call fb_set_ctrl takes rows [N][n_action] in the
 * environment's ACTION order; ctrl_index[c] is the ctrl slot of action c (-1: no actuator, e.g. a user action), NaN
 * actions are applied as 0 (tasks/base.py:197-201).  ctrl_index == NULL restores plain ctrl rows.                  */
int fb_set_action_map(FbHandle h, const int32_t* ctrl_index, int n_action);

/* walker.set_pose / set_velocity on a subset of coordinates (walk_imitation.py:141-145):
 * field in {FB_QPOS, FB_QVEL, FB_ACT, FB_QFRC_APPLIED, FB_XFRC_APPLIED}; vals is [N][k] AoS host (k <= 16), written to
 * coordinates idx[k] of every env.  No forward pass is run (dm_control does not run one either).                        */
int fb_write_state(FbHandle h, int field, const int32_t* idx, int k, const float* vals);
/* physics.data.qfrc_applied / physics.data.xfrc_applied in place, for a policy on the GPU: borrowed device pointers of the
 * compact rows [n_envs][nv] and [n_envs][nbody][6] (fp32, contiguous; allocated zeroed on first use, which any applied-force
 * call does).  Writes on another stream must be ordered before the next fb_step / fb_task_step on fb_stream.           */
int fb_applied_ptrs(FbHandle h, void** qfrc_applied_dev, void** xfrc_applied_dev);
/* Drop qfrc_applied and xfrc_applied of every env (mjData's are zero-filled; here the buffers are freed and the step goes
 * back to the path without the applied-force term).  Pointers of fb_applied_ptrs become invalid.                      */
int fb_clear_applied(FbHandle h);

/* Per-env model parameters: writes to physics.model without mj_setConst (what dm_control does), for every env of the batch on its
 * own.  Each parameter is named as its mjModel field; its size per env is fb_param_size (the step reads column 0 of geom_friction at
 * the model's condim <= 3, and entries 0 .. 2 of MuJoCo's ten gainprm / biasprm entries; all are stored).  Derived constants keep
 * their compiled values (body_invweight0, dof_invweight0, meaninertia, body_subtreemass, the task programs' constants); the
 * implicit-damping diagonal of the Euler step follows the env's dof_damping.  jnt_stiffness acts on hinge joints only, so the other
 * joints' entries must stay 0.
 *   The overlay [n_envs][parameters] is allocated on first use (fb_param_set / fb_param_draws) with every env at the compiled
 * values; it persists across steps and resets until overwritten or cleared (it is model, not data: resets do not restore it).
 * Allocating or clearing it drops the state bank (a state row then carries the env's parameters and draw counter) and
 * the captured step graphs.
 *   A draw program (fb_param_draws) redraws the listed parameters of an env at each of its resets (fb_reset, fb_reset_hold, a
 * device-task reset): lo + u (hi - lo) per element, u a counter hash of (seed, env, the env's draw count, parameter, element), or of
 * element 0 for every element of a `shared` parameter (one factor for all of them).  The same reset sequence gives the same rows
 * through the host-side and the device-side task code.
 *   Inputs are checked: parameter ids, sizes, env ids, finite values, no negative mass, inertia, armature, damping, stiffness,
 * friction, density or viscosity, lo <= hi.                                                                                        */
enum FbParam {
  FB_P_BODY_MASS = 0,        /* nbody                                                    */
  FB_P_BODY_INERTIA = 1,     /* nbody * 3 (principal inertia)                            */
  FB_P_DOF_ARMATURE = 2,     /* nv                                                       */
  FB_P_DOF_DAMPING = 3,      /* nv                                                       */
  FB_P_JNT_STIFFNESS = 4,    /* njnt                                                     */
  FB_P_GEOM_FRICTION = 5,    /* ngeom * 3                                                */
  FB_P_ACTUATOR_GAINPRM = 6, /* nu * 3                                                   */
  FB_P_ACTUATOR_BIASPRM = 7, /* nu * 3                                                   */
  FB_P_GRAVITY = 8,          /* 3 (mjModel.opt)                                          */
  FB_P_WIND = 9,             /* 3                                                        */
  FB_P_DENSITY = 10,         /* 1                                                        */
  FB_P_VISCOSITY = 11,       /* 1                                                        */
  FB_NPARAMS = 12
};
int fb_param_size(FbHandle h, int param);     /* values per env, -1 for an unknown id */
/* vals [n][size] (host, or device memory when is_device) -> the listed envs; env_ids NULL: every env, n must be n_envs. */
int fb_param_set(FbHandle h, int param, const int32_t* env_ids, int n, const float* vals, int is_device);
/* -> dst [n_envs][size] (host, or device memory when is_device); the compiled values while there is no overlay.  Synchronises. */
int fb_param_get(FbHandle h, int param, float* dst, int is_device);
/* Draw `param` at every reset from [lo, hi] ([size] host arrays each); shared != 0: one draw for all its elements.  NULL lo and hi
 * stop drawing it.  seed is the program's (every call sets it).                                                                  */
int fb_param_draws(FbHandle h, int param, const float* lo, const float* hi, int shared, uint32_t seed);
/* Free the overlay, the draw counters and the draw program: the step goes back to the compiled model's tables. */
int fb_param_clear(FbHandle h);

/* n_substeps x physics.step() with legacy_step=True, i.e. (mj_step2; mj_step1) per substep
 * (SURVEY.md App. A), accumulating the per-substep sensor mean.  Asynchronous on the handle's
 * stream.                                                                                     */
int fb_step(FbHandle h, int n_substeps);

/* mj_forward on all envs (after external state writes).                                       */
int fb_forward(FbHandle h);

/* Read a per-env field.  is_device=0: dst is host [N][n] AoS float32, synchronises.
 * is_device=1: *(void**)dst receives the borrowed device pointer of env 0's slots; consecutive envs
 * are fb_record_stride() 4-byte slots apart.                                                  */
int fb_get(FbHandle h, int field, void* dst, int is_device);
int fb_field_size(FbHandle h, int field);   /* floats per env, <0 on error */
int fb_record_stride(FbHandle h);           /* 4-byte slots between the records of consecutive envs */
int fb_set(FbHandle h, int field, const float* src);  /* host [N][n] AoS -> device, all envs */

/* Packed observation buffer of the last control step, [N][floats_per_env] AoS on device, for the
 * NCCL gather to rank 0 (SURVEY.md 8(e)).  Layout: qpos, qvel, act, sensor_mean, xpos/xmat of
 * root, site_xpos.                                                                            */
int fb_obs_ptr(FbHandle h, void** dev_ptr, int* floats_per_env);
/* Task observation program: the observables of the reference task (FruitFlyObservables, fruitfly.py:585-756;
 * ref_displacement / ref_root_quat, tasks/base.py:245-268) evaluated on the device right after fb_step, one
 * fp32 row per env in the task's final observation layout.  Items are concatenated in order.           */
enum FbObsItem {
  FB_OBS_SENSOR_MEAN = 0, /* a = sensordata adr, b = len : per-substep mean (first[e]: single sample / n_sub) */
  FB_OBS_SENSOR_NOW = 1,  /* a = adr, b = len           : last sample (termination checks)                   */
  FB_OBS_ACT = 2,         /* a = first act, b = len                                                          */
  FB_OBS_QPOS = 3,        /* a = offset into list, b = len : qpos[list[a..a+b)]                              */
  FB_OBS_QVEL = 4,
  FB_OBS_SITES_EGO = 5,   /* a = offset into list (site ids), b = count : (site_xpos - root_xpos) @ root_xmat */
  FB_OBS_ROOT_ZAXIS = 6,  /* root xmat[6:9]                                                                  */
  FB_OBS_REF_DISP = 7,    /* b = future_steps+1 : (ref_pos[step+i] - root_pos) @ root_xmat                   */
  FB_OBS_REF_QUAT = 8,    /* b = future_steps+1 : root_quat^-1 * ref_quat[step+i]                            */
  FB_OBS_SCALARS = 9,     /* flags, |qacc|^2, time                                                           */
  FB_OBS_ROOT_POSE = 10,  /* root xpos[3] + quat[4]                                                          */
  FB_OBS_SUBTREE_COM = 11,/* a = body id, 1 .. nbody - 1 (not the world) : physics.data.subtree_com[body]      */
  FB_OBS_DOF_AXIS_EGO = 12,/* a = offset into list (dof ids), b = count : world joint axis (physics.bind(joints).xaxis,
                              tasks/rewards.py:48-50) rotated into the root frame                                */
  FB_OBS_TASK_TARGET = 14,   /* b floats of the device task's per-episode targets (FB_TASK_VISION: target height, target speed = the reference's
                               `task_input` observable, tasks/vision_flight.py:56-76)                                     */
  FB_OBS_WORLD_CONTACT = 13 /* 1 float: 1 if an active contact (efc_address >= 0) involves a geom of the world body (ground plane, terrain):
                               the reference's check_floor_contact (tasks/vision_flight.py:235-247)                        */
};
typedef struct FbObsProgram {
  int32_t n_items; const int32_t* kind; const int32_t* a; const int32_t* b;
  int32_t n_list; const int32_t* list;
  int32_t root_body, n_sub;
  int32_t ref_len; const float* ref_qpos;      /* [ref_len][7] reference root trajectory */
} FbObsProgram;
/* Upload the program (and reference table); returns the row length in floats (<0 on error).             */
int fb_obs_program(FbHandle h, const FbObsProgram* p);
/* Per-env reference tables: every env tracks its own reference trajectory (one dataset snippet per episode, reference
 * tasks/walk_imitation.py:93-105, tasks/flight_imitation.py:88-106).  Called after fb_obs_program, fb_ref_slots switches
 * FB_OBS_REF_DISP / FB_OBS_REF_QUAT to a device table [n_envs][slot_len][7]; fb_ref_slot_write fills the slots of the
 * listed envs from rows [n][slot_len][7] (the caller pads a shorter snippet with its last row).  The step index given to
 * fb_task_inputs then counts inside the env's own slot.                                                  */
int fb_ref_slots(FbHandle h, int slot_len);
int fb_ref_slot_write(FbHandle h, const int32_t* env_ids, int n, const float* rows);
/* Per control step: index into the reference table and "first step after reset" flag of every env.      */
int fb_task_inputs(FbHandle h, const int32_t* step_idx, const uint8_t* first);
/* Copy the task observation rows [N][row_len] to a (pinned) host buffer (fb_pack_obs must have run).    */
int fb_read_task_obs(FbHandle h, float* host_dst);
/* Launch the pack kernel (after fb_step) / copy the packed rows to a (pinned) host buffer [N][floats_per_env]:
 * qpos, qvel, act, sensor_mean, sensordata, root xpos[3], root xmat[9], site_xpos[3*nsite], flags, |qacc|^2, time.
 * Stands in for the observation_updater reads of composer.Environment.step (SURVEY.md 3.3, R4).        */
int fb_pack_obs(FbHandle h);
int fb_read_obs(FbHandle h, float* host_dst);

/* Device-side task logic (SURVEY.md 8(f).2): everything the reference's task hooks do around the physics step -- composer
 * auto-reset + initialize_episode (tasks/walk_imitation.py:112-136, tasks/flight_imitation.py:113-144), before_step (ghost
 * placement walk_imitation.py:138-150; wing-beat pattern generator flight_imitation.py:146-168, pattern_generators.py:131-203),
 * check_termination / get_reward / get_discount (tasks/base.py:203-225, walk_imitation.py:179-203,
 * flight_imitation.py:170-226) -- evaluated on the device, so that a control step needs no host round trip: actions in
 * (host or device pointer), observation rows + (reward, discount, step_type) out.  Covers the shared-reference (inference-mode)
 * tasks and walk_imitation / flight_imitation with a trajectory dataset (FB_TASK_WALK / FB_TASK_FLIGHT with ref_bank = 1: fb_ref_slots, then
 * fb_ref_bank_wide / fb_ref_bank, then this program; every env draws its own trajectory (and, flight, start step) of the bank at
 * each reset).  Requires fb_set_action_map and fb_obs_program first.                                                 */
enum FbTaskKind {
  FB_TASK_WALK = 0,       /* walk_imitation */
  FB_TASK_FLIGHT = 1,     /* flight_imitation */
  FB_TASK_VISION = 2,     /* vision_guided_flight (fields at the end of FbTaskProgram) */
  FB_TASK_TEMPLATE = 3,   /* template_task (tasks/template_task.py): reset to reset_qpos at rest, no ghost / reference / before_step
                             hook; reward 1, LAST with discount 0 on a bad state or |qacc| > terminal_qacc, LAST with discount 1 at
                             time_limit (ghost_qadr = user_col = -1, no noise) */
  FB_TASK_BALL = 4        /* walk_on_ball (fields at the end of FbTaskProgram; FB_TASK_TEMPLATE's reset and hooks, its own reward) */
};
typedef struct FbTaskProgram {
  int32_t kind;                        /* enum FbTaskKind */
  int32_t root_qadr, root_vadr, ghost_qadr, ghost_vadr;   /* free-joint slots of the walker root and of the ghost (-1: none) */
  int32_t user_col;                    /* column of the beat-frequency action in the action row, -1 if none */
  float ghost_offset[3];
  float control_timestep, time_limit;
  float terminal_com_dist, terminal_linvel, terminal_angvel, terminal_qacc, terminal_height;
  int32_t velocimeter_adr, gyro_adr;   /* sensordata addresses */
  int32_t com_body;                    /* body whose subtree CoM the flight reward tracks */
  int32_t episode_steps;               /* step index that ends the episode (end of the reference) */
  int32_t ref_len; const float* ref_qpos /* [ref_len][7] */; const float* ref_qvel /* [ref_len][6] */;
  int32_t obs_refdisp_off, obs_refquat_off;   /* offsets of ref_displacement / ref_root_quat inside the observation row */
  const float* reset_qpos;             /* [nq] episode start pose (root / ghost slots are overwritten from the reference) */
  int32_t n_noise; const int32_t* noise_qadr; float noise_amp; uint32_t seed;   /* U(-amp, amp) on these qpos at reset */
  int32_t n_wing; const int32_t* wing_qadr; const int32_t* wing_vadr; const int32_t* wing_ctrl;
  int32_t n_freq, tab_len;             /* wing-beat tables: one resampled pattern per discrete beat frequency */
  const float* wb_traj /* [n_freq][tab_len][n_wing] */; const float* wb_phase; const float* wb_phase_mod /* [n_freq][tab_len], +inf padded */;
  const float* wb_freqs /* [n_freq] */; const int32_t* wb_len /* [n_freq] */;
  float wb_base_freq, wb_rel_range, wb_rate;
  float com_offset[3];                 /* root -> CoM offset in the root frame (tasks/task_utils.py:237) */
  /* FB_TASK_VISION, vision_guided_flight (tasks/vision_flight.py:97-254): no ghost / reference; per episode a target height and speed, a start
   * point, a wing-beat phase and a terrain of the device bank (fb_hfield_bank) are drawn; reward = product of the height / forward speed /
   * speed / side speed / body axis factors and, for 'trench' arenas, the distance to the corridor's centre line (vision_flight.py:214-226:
   * y of the centre line at trench_len[k] equally spaced x in [trench_x[k][0], trench_x[k][1]] for bank terrain k);
   * termination on a bad state or, if floor_contacts_fatal, an active contact with a world geom.                                */
  float target_height_range[2], target_speed_range[2], init_x_range[2], init_y_range[2];
  float hover_quat[4], target_zaxis[3];
  int32_t floor_contacts_fatal;
  int32_t trench_cap;                  /* 0: no centre-line factor; else the row stride of trench_y */
  const float* trench_x /* [n_terrain][2] first / last x */; const int32_t* trench_len /* [n_terrain] samples */; const float* trench_y /* [n_terrain][trench_cap] */;
  /* FB_TASK_FLIGHT with a trajectory dataset (tasks/flight_imitation.py:88-111, trajectory_loaders.py:67-141).  ref_bank = 1: per-env
   * references from the bank of fb_ref_bank, written into the env's fb_ref_slots table at each reset (ref_qpos / ref_qvel /
   * episode_steps are then unused).  A reset takes the pick pinned by fb_task_ref_pick, else draws from the counter hash: the
   * trajectory uniformly over pick_traj (repeats allowed), the start step uniformly in [0, len - start_margin) if
   * randomize_start, else 0.  Rows in use n = min(len - start, slot_len); the episode ends at step
   * min(n, max_episode_rows) - (future_steps + 1).  Zero (the default of a zeroed struct): shared reference.           */
  int32_t ref_bank;
  int32_t n_pick; const int32_t* pick_traj /* [n_pick] trajectory indices of the bank */;
  int32_t randomize_start, start_margin;
  int32_t max_episode_rows;            /* flight: round(time_limit / control_timestep); walking: max_episode_steps + future_steps + 1 */
  int32_t future_steps;
  /* FB_TASK_WALK with a trajectory dataset (tasks/walk_imitation.py:93-177): ref_bank = 1 with a bank of fb_ref_bank_wide whose rows are
   * 15 + 6 n_mocap_joints + 3 n_mocap_sites wide; randomize_start = 0 (every snippet starts at row 0).  A reset puts the root and
   * ghost on row 0 (root x, y shifted to the origin), the mocap joints at the snippet's row-0 qpos, the wings back at wing_spring,
   * then adds the noise.  The reward is the product of the four DeepMimic factors
   * deep_mimic_weight[k] * exp(-0.5 / deep_mimic_std[k]^2 * diff_k) (com, qvel, root2site, joint_quat; tasks/rewards.py:86-116) and
   * the n_wing factors max(0, 1 - |wing qpos - wing_spring| / retract_margin), from the walker features in the observation
   * row (obs_*_off: root pose 7, root qvel 6, mocap qpos nj, mocap qvel nj, mocap joint axes nj x 3, mocap sites ns x 3, wing qpos
   * n_wing) and the bank row of step min(step, n - 1).  wing_qadr / n_wing name the wing joints.  Zero: no such fields.  */
  int32_t n_mocap_joints; const int32_t* mocap_qadr /* [n_mocap_joints] */; int32_t n_mocap_sites;
  int32_t obs_root_pose_off, obs_root_qvel_off, obs_mocap_qpos_off, obs_mocap_qvel_off, obs_mocap_axes_off, obs_mocap_sites_off, obs_wing_qpos_off;
  const float* wing_spring;            /* [n_wing] */
  float deep_mimic_std[4], deep_mimic_weight[4], retract_margin;
  /* FB_TASK_BALL, walk_on_ball (tasks/walk_on_ball.py:55-81): the reset is FB_TASK_TEMPLATE's (reset_qpos at rest); the reward is the product over
   * i < 3 of max(0, 1 - |qvel[ball_vadr + i] - ball_target[i]| / ball_margin); an episode ends with discount 0 when |velocimeter| >
   * terminal_linvel, |gyro| > terminal_angvel or the state is bad, and with discount 1 at the time limit.  */
  int32_t ball_vadr; float ball_target[3], ball_margin;
} FbTaskProgram;
int fb_task_program(FbHandle h, const FbTaskProgram* p);
/* Flight trajectory bank for FB_TASK_FLIGHT with ref_bank: n_traj trajectories, rows [sum(traj_len)][15] fp32, trajectory k after
 * trajectory k - 1: root qpos (7; the dataset's CoM pose through com2root), CoM qvel (6), CoM x, y (2).  A reset at start step s
 * shifts the root x, y of its rows by the CoM x, y of row s (every episode starts above the origin, trajectory_loaders.py:120).
 * Uploaded once; calling it again replaces the bank and drops a task program that points at it.  = fb_ref_bank_wide(.., 15, ..) */
int fb_ref_bank(FbHandle h, int n_traj, const int32_t* traj_len, const float* rows);
/* Trajectory bank with rows of row_width >= 15 floats; the first 15 columns keep their flight meaning (columns 13, 14: the x, y a
 * reset at that row shifts the root x, y by).  Walking (FB_TASK_WALK): root qpos 7, root qvel 6, root x, y 2, then mocap qpos [nj],
 * mocap qvel [nj], root2site [ns][3], joint_quat [nj][4] of the dataset (trajectory_loaders.py:146-156).  At most 2^31 - 1 rows in
 * all; a bank larger than the device's free memory is refused (-4) with an fb_last_error message.                      */
int fb_ref_bank_wide(FbHandle h, int n_traj, const int32_t* traj_len, int row_width, const float* rows);
/* Pin the trajectory and start step of the listed envs' next reset (consumed and cleared by that reset) -- the draws of a host
 * RandomState, where the counter hash would draw otherwise.  Needs a program with ref_bank.                           */
int fb_task_ref_pick(FbHandle h, const int32_t* env_ids, int n, const int32_t* traj, const int32_t* start);
/* Trajectory and start step of every env's running episode, int32 [n_envs] each, to the host (synchronises).          */
int fb_task_ref_state(FbHandle h, int32_t* traj, int32_t* start);
/* One control step with the task logic on the device: [auto-reset] -> action -> ctrl -> before_step -> n_substeps x physics ->
 * observation program -> termination / reward.  `action` rows [n_envs][n_action] (fb_set_action_map), host or device.  */
int fb_task_step(FbHandle h, const float* action, int is_device, int n_substeps);
/* Mark every env for reset at the next fb_task_step (env.reset()).                                                    */
int fb_task_reset_all(FbHandle h);
/* Amplitude of the U(-a, a) joint noise the device-side reset adds to the listed start-pose joints (FbTaskProgram.noise_amp), changed
 * without re-uploading the program: e.g. noise for the very first reset only (decorrelated start states), exact start pose at the
 * auto-resets, as the reference's initialize_episode has it.                                                            */
int fb_task_set_reset_noise(FbHandle h, float amp);
/* Mark the listed envs for reset at the next fb_task_step, whatever their episode state (an actor restarting single
 * environments; bench.py's pre-roll uses it to spread the envs over the phases of an episode).                          */
int fb_task_request_reset(FbHandle h, const int32_t* env_ids, int n);
/* Per-env count of episodes started so far (resets done by the device-side task logic), int32 [n_envs] to the host.    */
int fb_task_episodes(FbHandle h, int32_t* dst);
/* Terrain bank for the device-side vision task: K heightfields [K][nrow * ncol] (heights as fb_hfield_write takes them, the grid
 * of fb_hfield_collision / fb_eye_program); a resetting env copies one of them into its own heightfield (collision + eyes).  */
int fb_hfield_bank(FbHandle h, int n_terrain, const float* heights);
/* Rows of 8 uniform numbers in [0,1) consumed by the listed envs' next reset instead of the device's counter hash (FB_TASK_VISION:
 * target height, target speed, start x, start y, wing-beat phase, terrain pick; FB_TASK_FLIGHT: wing-beat phase) -- lets a test feed the device the
 * draws of the host-side task code.                                                                                    */
int fb_task_uniform_rows(FbHandle h, const int32_t* env_ids, int n, const float* u);
/* Uniform numbers in [0,1) consumed by the listed envs' next reset (flight: wing-beat phase); without them the device
 * draws from a counter hash of (seed, env, episode).                                                                 */
int fb_task_uniforms(FbHandle h, const int32_t* env_ids, int n, const float* u);
/* Results of the last fb_task_step: borrowed device pointers (obs rows [n_envs][obs_dim], out rows [n_envs][4] = reward,
 * discount, step_type 0 FIRST / 1 MID / 2 LAST, 0) and the host copy (synchronises).                                  */
int fb_task_ptrs(FbHandle h, void** obs_dev, int* obs_dim, void** out_dev);
int fb_task_read(FbHandle h, float* obs_host, float* out_host);
/* Eye cameras (reference FruitFlyObservables.right_eye / left_eye, fruitfly/fruitfly.py:729-745; cameras fruitfly.xml:335-336;
 * 32 x 32 RGB, fovy 150 deg in tasks/vision_flight.py:23-24): a ray caster over a per-env heightfield terrain
 * (tasks/arenas/hills.py), the ground plane and a sky, from the current body poses.  MuJoCo's camera model (pinhole, -z forward,
 * +y up, vertical fovy, row 0 at the top); not MuJoCo's OpenGL image.                                                  */
typedef struct FbEyeProgram {
  int32_t n_cam;                         /* 1 or 2 */
  int32_t body[2]; float pos[2][3]; float quat[2][4];   /* camera frames in the frame of the body they are attached to */
  float fovy_deg; int32_t size;          /* vertical field of view; images are size x size */
  int32_t nrow, ncol; float half_size;   /* heightfield grid over [-half_size, half_size]^2 (row = y, col = x); nrow = 0: none */
  float z_offset, zfar;                  /* height of the ground plane / terrain base (hills.py:210), far clipping distance */
  float sky_top[3], sky_horizon[3], ground[3], ambient, diffuse;   /* colours in [0,1]; headlight terms (hills.py:248-250) */
} FbEyeProgram;
int fb_eye_program(FbHandle h, const FbEyeProgram* p);
/* Heightfield collision (MuJoCo mjc_ConvexHField; the terrain of tasks/arenas/hills.py): `geom` is the model's heightfield geom
 * (pose and contact parameters come from the model; any pose), size = (x half extent, y half extent, elevation scale, base depth),
 * the grid is nrow x ncol, pair_geom lists the 1 .. 192 (FB_MAXCAND) geoms that can touch it (repeats allowed), up to 4 contacts
 * each.  Adds one kernel between collision and constraint rows.  The per-env heights h are the ones of fb_hfield_write (shared
 * with the eye cameras): the surface lies h * size[2] above the terrain geom's frame.                                       */
int fb_hfield_collision(FbHandle h, int geom, const float* size, int nrow, int ncol, const int32_t* pair_geom, int npair);
/* Heights h of the listed envs' terrains, rows [n][nrow * ncol]; envs never written are flat.  The collision stage scales them
 * by the elevation scale size[2] of fb_hfield_collision (1 for the `vision` model, where h is in world units).             */
int fb_hfield_write(FbHandle h, const int32_t* env_ids, int n, const float* heights);
/* Render every env's eyes from the current poses into the library's buffer [n_envs][n_cam][size][size][3] (uint8).   */
int fb_render_eyes(FbHandle h);
/* The device address of that buffer and its bytes per env.  The pointer is valid until the next fb_eye_program, which frees the
 * buffer and allocates a new one, or fb_destroy.                                                                         */
int fb_eyes_ptr(FbHandle h, void** dev_ptr, int* bytes_per_env);
int fb_eyes_read(FbHandle h, uint8_t* host_dst);
/* State rows: the batched stand-in for physics.get_state() / physics.set_state() (dm_control), extended by what a batched
 * task env carries per env.  A row is everything the next fb_step / fb_task_step of an env reads that the position / velocity
 * stage does not recompute from it: qpos, qvel, act, ctrl, qacc, time, flags, solver iterations, hold, the solver's warm start
 * (previous row keys, count, forces), sensordata and the per-step sensor sums, the env's packed and task observation rows with
 * their step index / FIRST flag, its reference slot (fb_ref_slots), its applied forces if the handle has them, its model parameters
 * and draw counter if the handle has a parameter overlay (fb_param_set), and the device
 * task's per-env arrays (counters, reset flags, staged draws, wing-beat generator, `out` row, dataset episode and pin, vision
 * targets and terrain pick).  A rollout continued from a loaded row equals the uninterrupted one bit for bit.
 *   After fb_state_load, fb_get returns the saved values for the fields above and freshly recomputed ones for everything the
 * position / velocity stage writes (FB_XPOS .. FB_SITE_XMAT, FB_SUBTREE_COM, FB_QM_DENSE, FB_NCON, FB_NEFC, FB_CONTACT,
 * FB_QFRC_BIAS, FB_QFRC_PASSIVE); the acceleration stage's leftovers (FB_QFRC_SMOOTH, FB_QFRC_CONSTRAINT, FB_QFRC_ACTUATOR,
 * FB_EFC_FORCE) keep what the env held before the load until the next step rewrites them.  Terrains are not in the row: the
 * device vision task copies the row's terrain of its bank when the env holds another one, terrains written by
 * fb_hfield_write are the caller's to rewrite.  The device task's draws are a counter hash of (seed, env, episode): a row
 * loaded into another env id continues bit for bit until that env's next reset, whose draws follow the new id.
 *   The layout follows the handle: replacing the observation or task program, the reference slots, a bank a task program draws
 * from, or allocating / clearing the applied-force arrays or the parameter overlay drops the bank, and save / load fail with a message until
 * fb_state_bank is called again.  fb_state_signature hashes the layout (sizes, program kinds, slot length, layout version);
 * rows move between handles with equal signatures.  Saving and loading change nothing a captured step graph depends on.    */
int fb_state_slots(FbHandle h);                  /* 4-byte slots of one row under the handle's current model, programs and applied-force arrays */
uint64_t fb_state_signature(FbHandle h);
int fb_state_bank(FbHandle h, int n_slots);      /* (re)allocate the device bank [n_slots][fb_state_slots]; 0 frees it; -4 with a message if it does not fit */
/* env_ids[k] -> slots[k], stream-ordered (no synchronisation); a NULL list is the identity 0 .. n - 1, both NULL: every env k -> slot k.
 * A slot may be written once per call.                                                                                       */
int fb_state_save(FbHandle h, const int32_t* env_ids, const int32_t* slots, int n);
/* slots[k] -> env_ids[k], then the position / velocity stage of the loaded envs only; the other envs are untouched.  One slot may
 * feed many envs, an env may appear once.  A row saved while envs were held for their reset makes the next step a holding one.  */
int fb_state_load(FbHandle h, const int32_t* slots, const int32_t* env_ids, int n);
int fb_state_read(FbHandle h, const int32_t* slots, int n, void* host_dst);          /* bank rows -> host [n][fb_state_slots], synchronises */
int fb_state_write(FbHandle h, const int32_t* slots, int n, const void* host_src);   /* host rows -> bank */
/* The one handle-level number a continuation on another handle needs: the substeps of the last fb_step (the divisor of the per-step
 * sensor means).  Returns it; n_substeps > 0 sets it first (a handle that never stepped continuing another one's rows).        */
int fb_state_substeps(FbHandle h, int n_substeps);
/* Multi-site inverse kinematics (reference flybody/inverse_kinematics.py: qpos_from_site_xpos), one problem per env, one warp each.
 * Gradient descent with momentum on  sum over included components of (site_xpos - target)^2 + reg_strength * |hinge qpos|^2  (the
 * fitted hinges' raw qpos, as the reference), the step applied as mj_integratePos; every 100 iterations (from iteration 0) the
 * objective is evaluated and the problem stops with success when lr |u| / objective < progress_threshold (an objective of 0 counts
 * as converged: the reference divides by it).  Fitted joints are hinge or free joints; ball joints cannot be fitted, unfitted ones
 * keep their qpos.  The program owns its buffers; the record layout, the state rows and fb_state_signature do not change.   */
typedef struct FbIkProgram {
  int32_t n_sites; const int32_t* site_ids;    /* model site ids, 1 .. 64 of them                                         */
  int32_t n_jnts; const int32_t* jnt_ids;      /* fitted joints (hinge or free), each once                                 */
  const uint8_t* include;                      /* [3 * n_sites] components in the objective (include_inds); NULL = all      */
  float reg_strength, lr, beta, progress_threshold;
  int32_t max_steps;                           /* >= 1                                                                      */
} FbIkProgram;
int fb_ik_program(FbHandle h, const FbIkProgram* p);
/* Envs 0 .. n-1: qpos <- init_qpos rows [n][nq] (NULL: keep the current qpos), then solve for targets [n][n_sites][3] (world frame).
 * A NaN target component is excluded for that problem (a tracking dropout); an infinite target or a non-finite init_qpos is an
 * error.  Runs bounded launches on the handle's stream and reads one live count per launch, so it returns when every problem has
 * stopped.  Afterwards qpos holds the fits; the other forward quantities are stale until fb_forward / fb_reset.             */
int fb_ik_solve(FbHandle h, int n, const float* target_xpos, const float* init_qpos);
/* Results of the last solve for its n problems, each pointer may be NULL (synchronises): qpos [n][nq]; err: the objective at the
 * last check; err_first: the site term at the returned qpos; steps: the loop index at the stop (max_steps - 1 without success);
 * success: 1 when the progress test stopped the problem.                                                                   */
int fb_ik_read(FbHandle h, float* qpos, float* err, float* err_first, int32_t* steps, uint8_t* success);
/* Inverse dynamics (MuJoCo mj_inverse, continuous time; dm_control `mjlib.mj_inverse` then `data.qfrc_inverse`, `data.efc_force`):
 * the forces that give envs 0 .. n-1 the accelerations qacc [n][nv] (host rows, or a device pointer on the handle's stream when
 * is_device) at their current qpos, qvel and act.  Runs the position / velocity stage of every env (the launches fb_forward starts
 * with, without sensor sums), then one inverse kernel; it writes nothing else into the record, so on a current state (after fb_reset,
 * fb_forward or fb_step) the record is bit for bit unchanged and the next fb_step is too.  Per problem:
 *   efc_force       = the soft constraint model's forces at jar = J qacc - aref, aref = -B J qvel - K imp (pos - margin)
 *                     (mj_constraintUpdate: limits, frictionless and elliptic contacts);
 *   qfrc_constraint = J^T efc_force;  qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint.
 * qfrc_inverse excludes applied and actuator forces: for the continuous-time qacc fb_forward leaves in FB_QACC it equals
 * qfrc_applied + J^T xfrc_applied + qfrc_actuator up to the forward solve's tolerance.  Noslip is not inverted (as in MuJoCo): on a
 * model with noslip iterations the forces are the soft model's, not the forward step's post-noslip friction.  The discrete inverse
 * (mjENBL_INVDISCRETE) is not implemented.  Problem i runs in env i, so with a parameter overlay (fb_param_set) it uses env i's
 * model parameters.  Errors: n outside 1 .. n_envs, a NULL qacc, a non-finite host qacc.  A device qacc is
 * not checked and the call returns without synchronising; with a host qacc it synchronises.                                    */
int fb_inverse(FbHandle h, int n, const float* qacc, int is_device);
/* Results of the last fb_inverse for its n problems (synchronises; any pointer may be NULL; is_device: the pointers are device
 * memory): qfrc_inverse [n][nv], qfrc_constraint [n][nv], efc_force [n][fb_field_size(FB_EFC_FORCE)], rows as FB_CONTACT's efc_adr
 * and FB_NEFC index them after the call (rows >= nefc hold 0).  An error before the first fb_inverse.                         */
int fb_inverse_read(FbHandle h, float* qfrc_inverse, float* qfrc_constraint, float* efc_force, int is_device);
/* Finite-difference transition Jacobians (MuJoCo mjd_transitionFD; C and D: fb_query_sensors; dm_control `mjlib.mjd_transitionFD`):
 *   A [nx][nx] = dx'/dx and B [nx][nu] = dx'/du, row-major as MuJoCo's, x = (dq [nv], qvel [nv], act [na]) with dq the tangent of qpos
 *   (mj_integratePos to nudge, mj_differentiatePos to difference), nx = 2 nv + na, u = ctrl [nu];
 *   x' = the state after n_substeps substeps (mj_step2; mj_step1: fb_step's launches) with ctrl held fixed; n_substeps = 1 is
 *   mjd_transitionFD, the task's substep count the transition of one control step.
 * A problem is a state row of the bank (fb_state_save / fb_state_write).  It takes fb_fd_columns(h, centered) envs: 1 + 2 (nx + nu)
 * centred, 1 + nx + nu forward; column 0 is the unperturbed nominal.  Every column starts from the row, its warm start included (as
 * MuJoCo restores qacc_warmstart before each nudged step), and from its applied forces when the rows carry them (held fixed, as
 * mjData's are), and from its model parameters when the rows carry an overlay (fb_param_set).  Coordinate j is nudged by delta_j = eps max(1, |x_j|) (x_j: the hinge angle, the free joint's translation component,
 * qvel, act or ctrl; rotational tangent coordinates delta = eps): the stepper is fp32, and a step relative to the coordinate keeps fast
 * ones resolved (MuJoCo's absolute step is the case |x_j| <= 1; flybody_b200.derivatives defaults to eps 1e-2).  ctrl at its limits follows MuJoCo: forward if the actuator is not
 * ctrl-limited or ctrl and ctrl + delta lie in its range, backward if (centred or no forward nudge) and ctrl - delta and ctrl do;
 * centred, one-sided or a zero column.
 * fb_fd_transition runs problems slots[0 .. n-1] (host ints) on envs k ncol .. (k+1) ncol - 1; the envs past n ncol run copies of the
 * last problem.  The handle is a workspace: afterwards every env's state is unspecified; the bank is untouched.  Errors: no bank, a slot
 * out of range, never written or saved while its env was held for a reset, n < 1 or n ncol > n_envs, eps <= 0 or not finite,
 * n_substeps < 1.  It synchronises.                                                                                                  */
int fb_fd_columns(FbHandle h, int centered);
int fb_fd_transition(FbHandle h, const int32_t* slots, int n, float eps, int centered, int n_substeps);
/* Results of the last fb_fd_transition for its n problems (synchronises; any pointer may be NULL; is_device: the pointers are device
 * memory): A [n][nx][nx], B [n][nx][nu], and the nominal column's next state qpos_next [n][nq], qvel_next [n][nv], act_next [n][na].
 * An error before the first fb_fd_transition.                                                                                        */
int fb_fd_read(FbHandle h, float* A, float* B, float* qpos_next, float* qvel_next, float* act_next, int is_device);
/* Finite-difference inverse-dynamics Jacobians (MuJoCo mjd_inverseFD with flg_actuation = 0; DsD*: fb_query_sensors): the derivatives of
 * fb_inverse's qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint, and of qM, with respect to the inputs
 * (dq [nv], qvel [nv], qacc [nv]), dq the tangent of qpos (mj_integratePos to nudge).  The outputs are TRANSPOSED, as MuJoCo's
 * ("all outputs are transposed"), and so the transpose of fb_fd_transition's row-major A and B: row i is the derivative with respect
 * to input i,
 *   DfDq [nv][nv], DfDv [nv][nv], DfDa [nv][nv]  with DfDq[i][j] = d qfrc_inverse_j / d dq_i;
 *   DmDq [nv][nM]  d qM / d dq_i in MuJoCo's sparse qM order (the diagonal at dof_Madr, then the ancestors).
 * A problem is one state (qpos [nq], qvel [nv], qacc [nv]) and takes fb_fd_inverse_columns(h, centered) envs: 1 + 2 (3 nv) centred,
 * 1 + 3 nv forward (MuJoCo's mjd_inverseFD is forward-only); column 0 is the nominal.  The columns and step are fb_fd_transition's:
 * input j is nudged by delta_j = eps max(1, |x_j|) (x_j: the hinge angle, the free joint's translation component, qvel or qacc;
 * rotational tangent coordinates delta = eps).  flybody_b200.derivatives defaults to eps 1e-2.
 * fb_fd_inverse runs problems qpos [n][nq], qvel [n][nv], qacc [n][nv] (host rows, or device pointers on the handle's stream when
 * is_device) on envs k ncol .. (k+1) ncol - 1; the envs past n ncol hold copies of the last problem.  Every env runs the position /
 * velocity stage (as fb_inverse), then the inverse kernel.  Each env's other inputs (act, ctrl, applied forces) are whatever it
 * holds; none of them reaches qfrc_inverse.  The handle is a workspace: afterwards every env's qpos / qvel and the record are
 * unspecified; fb_inverse_read still returns the last fb_inverse and the state bank is untouched.  Noslip is not inverted (as in
 * fb_inverse and MuJoCo): on a model with noslip iterations the forces are the soft model's.  Errors: n < 1 or n ncol > n_envs, a
 * NULL input, a non-finite host input, eps <= 0 or not finite, a parameter overlay on the handle (the columns are written from
 * qpos, qvel and qacc alone and would run with the parameters of whichever env they land in: fb_param_clear first).  A device input is not checked and the call returns without
 * synchronising; with host inputs it synchronises.                                                                                   */
int fb_fd_inverse_columns(FbHandle h, int centered);
int fb_fd_inverse(FbHandle h, int n, const float* qpos, const float* qvel, const float* qacc, float eps, int centered, int is_device);
/* Results of the last fb_fd_inverse for its n problems (synchronises; any pointer may be NULL; is_device: the pointers are device
 * memory): DfDq, DfDv, DfDa [n][nv][nv], DmDq [n][nv][nM] and the nominal column's qfrc_inverse [n][nv].  An error before the first
 * fb_fd_inverse.                                                                                                                     */
int fb_fd_inverse_read(FbHandle h, float* DfDq, float* DfDv, float* DfDa, float* DmDq, float* qfrc_inverse, int is_device);
/* Sensors in the dynamics queries.  While fb_query_sensors(h, 1) is on, fb_inverse, fb_fd_transition and fb_fd_inverse also produce
 * sensor outputs, columns in the model's sensor_adr order (nsd = nsensordata); while it is off (the default) they launch exactly the
 * kernels they launch without it.  Either way their other outputs, the record after fb_inverse and the state bank are bit for bit
 * the same.  Its buffers are allocated on the first call with sensors on.  A model with nsensordata = 0 launches nothing more and
 * reads empty outputs.  Errors: a model whose sensor pass (18 floats per body per warp) does not fit in shared memory.
 *   fb_inverse:       sensordata [n][nsd] as MuJoCo's mj_inverse evaluates it: gyro and velocimeter of the state; accelerometer,
 *                     force and touch of the finish kernel's sensor pass at the given qacc and the inverse's efc_force (touch: the
 *                     normal forces of the contacts whose ray hits the site volume).  As in the step, xfrc_applied does not enter
 *                     the force sensors (MuJoCo's cfrc_ext has it); on a noslip model touch and force are the soft model's.
 *   fb_fd_transition: C [n][nsd][nx] = ds/dx and D [n][nsd][nu] = ds/du, row-major as A and B, s the sensors of x, the state before
 *                     the step (MuJoCo's mjd_transitionFD), for any n_substeps: not the substep mean a policy observes.  The first
 *                     substep is launched on its own (the same launches), and the nominal sensordata [n][nsd] is that of x.
 *   fb_fd_inverse:    DsDq, DsDv, DsDa [n][nv][nsd], transposed as DfD* (DsDq[i][k] = d sensordata_k / d dq_i), of the inverse's
 *                     sensordata, and the nominal column's sensordata [n][nsd].                                              */
int fb_query_sensors(FbHandle h, int on);
/* The sensor outputs of the last call of each query (synchronises; any pointer may be NULL; is_device: the pointers are device memory).
 * Errors: a read before any call of the query, a read after a call made with sensors off.                                      */
int fb_inverse_sensor_read(FbHandle h, float* sensordata, int is_device);
int fb_fd_sensor_read(FbHandle h, float* C, float* D, float* sensordata, int is_device);
int fb_fd_inverse_sensor_read(FbHandle h, float* DsDq, float* DsDv, float* DsDa, float* sensordata, int is_device);
/* Finite-difference parameter Jacobians (system identification): the derivatives of fb_fd_transition's next state and of
 * fb_inverse's qfrc_inverse (and of their sensors while fb_query_sensors is on) with respect to directions in the per-env model
 * parameters (fb_param_*).  Derived constants hold as in the overlay (no mj_setConst); the implicit-damping diagonal follows dof_damping.
 *   A direction program (fb_fd_param_program) lists k >= 1 directions; direction j has the entries dir_ptr[j] .. dir_ptr[j+1] - 1 of
 *   param[] (FbParam ids) and elem[] (elements as fb_param_size counts them):
 *     kind 0, element: one entry theta_i, nudged by +-delta_i = eps max(|theta_i|, floor_i), theta_i the problem's own value; the column
 *                      is d / d theta_i in the parameter's units.  A side whose value would be negative on a non-negative field (those
 *                      fb_param_set keeps >= 0) is skipped, as fb_fd_transition skips a ctrl nudge out of range: a one-sided column.
 *     kind 1, scale:   every entry multiplied by (1 +- eps); the column is d / ds at s = 1 of theta_set <- s theta_set.  Needs eps < 1.
 *   floor[] is read for element entries only (positive, finite).  Errors: k < 0, NULL arrays, dir_ptr not starting at 0 or not
 *   increasing, an unknown kind or parameter, an element out of range, an element direction of more than one entry, jnt_stiffness of
 *   a joint that is not a hinge, an element twice in one direction.  k = 0 clears the program.  fb_fd_param_columns(h, centered): the
 *   envs of one problem, 1 + 2k centred, 1 + k forward (column 0 the nominal); -1 without a program.
 * Both queries need a parameter overlay (fb_param_set) and a program; eps > 0 and finite.  The handle is a workspace: afterwards every
 * env's state and parameters are unspecified (the overlay rows of the columns hold their nudged values); the bank is untouched.
 *   fb_fd_param_transition: fb_fd_transition's contract (problems are state-bank rows, which carry the parameters; columns fanned out
 *     and stepped n_substeps substeps with ctrl held; the same errors).  Outputs (fb_fd_param_read): dxdp [n][nx][k] row-major as B
 *     (mj_differentiatePos rows for dq), the nominal next state; with sensors (fb_fd_param_sensor_read): dsdp [n][nsd][k] and the
 *     nominal sensordata, the sensors of x, the state before the step (as C and D).  It synchronises.
 *   fb_fd_param_inverse: problems qpos [n][nq], qvel [n][nv], qacc [n][nv] (host rows, or device pointers when is_device) as
 *     fb_fd_inverse; problem i takes env i's parameter row at call time (as fb_inverse).  Outputs (fb_fd_param_inverse_read):
 *     DfDp [n][k][nv] transposed as DfDq (DfDp[j][i] = d qfrc_inverse_i / d direction j), the nominal qfrc_inverse; with sensors
 *     (fb_fd_param_inverse_sensor_read): DsDp [n][k][nsd] and the nominal sensordata.  qfrc_inverse excludes actuation, so actuator
 *     gain / bias columns are 0.  Errors: fb_fd_inverse's.  A device input is not checked and the call does not synchronise.
 * The reads synchronise (any pointer may be NULL; is_device: device pointers).  Errors: a read before any call, a sensor read after a
 * call made with sensors off.                                                                                                        */
int fb_fd_param_program(FbHandle h, int k, const int32_t* kind, const int32_t* dir_ptr, const int32_t* param, const int32_t* elem, const float* floor);
int fb_fd_param_columns(FbHandle h, int centered);
int fb_fd_param_transition(FbHandle h, const int32_t* slots, int n, float eps, int centered, int n_substeps);
int fb_fd_param_read(FbHandle h, float* dxdp, float* qpos_next, float* qvel_next, float* act_next, int is_device);
int fb_fd_param_sensor_read(FbHandle h, float* dsdp, float* sensordata, int is_device);
int fb_fd_param_inverse(FbHandle h, int n, const float* qpos, const float* qvel, const float* qacc, float eps, int centered, int is_device);
int fb_fd_param_inverse_read(FbHandle h, float* DfDp, float* qfrc_inverse, int is_device);
int fb_fd_param_inverse_sensor_read(FbHandle h, float* DsDp, float* sensordata, int is_device);
/* Batched rollouts (MuJoCo's mujoco.rollout.rollout, and the host loop of set_control, step and field reads it replaces): n rollouts
 * of T control steps, each step n_substeps substeps (mj_step2; mj_step1) with ctrl held over them.  Rollout i runs in env i from
 * state-bank row slots[i] (slots may repeat: K rollouts from one state); envs n .. n_envs-1 run a copy of the last rollout, whose
 * outputs are not written (the transition query's fan-out).  Each control step is an input kernel, the step graph fb_step replays and
 * a record kernel: no host synchronisation or copy inside the horizon, and no change to the step kernels.  Afterwards the envs are a
 * workspace (their state is that of the rollouts' last step); the bank and the other queries' results are untouched.
 *   Inputs (host rows, or device pointers when is_device): ctrl [n][T][nu]; step t writes row t into d->ctrl before its first substep,
 *   unclamped (the actuation stage clamps ctrl-limited actuators, as it does for d->ctrl).  qfrc_applied [n][T][nv] and xfrc_applied
 *   [n][T][nbody][6] (either may be NULL) are written the same way (MuJoCo rollout's control_spec for applied forces); without them the
 *   row's applied forces persist.  They need the applied-force arrays (fb_applied_ptrs) before the bank is laid out.
 *   Feedback (fb_rollout_feedback, set once for the calls that follow; T = 0 or both NULL clears it): nominal states xref
 *   [T][nq + nv + na] and gains K [T][nu][nx], nx = 2 nv + na, shared by every rollout.  Step t writes ctrl = u_t + K_t (x_t - xref_t),
 *   x_t the state the step starts from and the difference fb_fd_transition's tangent (mj_differentiatePos(xref qpos, qpos) per joint,
 *   then qvel and act), so gains from a Riccati recursion on its A and B apply without conversion.  Fixed order: a rollout's bits do
 *   not depend on its slot or on the batch size.
 *   A bank of laws (fb_rollout_feedback_bank, in place of the shared law): xref [L][T][nq + nv + na] and K [L][T][nu][nx] (fp32, host
 *   rows or device pointers as is_device says), and the host list law [n] (int32, values in [0, L)): rollout i applies law law[i], with
 *   the same arithmetic as the shared law, so its bits equal a shared-law call with that law.  The fb_rollout calls that follow must
 *   have n rollouts.  fb_rollout_feedback is the bank of L = 1 without a list (any n).  The buffers are kept and grown on use; -4 with
 *   a message when they do not fit.  Errors: fb_rollout_feedback's, L < 1, L > 1 without a list, a list of n < 1, a law out of range;
 *   it synchronises with host arrays or a list.
 *   Records (fb_rollout_read), after control step t in row [i][t]: qpos [n][T][nq], qvel, act, ctrl as written, time [n][T] and the
 *   env's flags [n][T].  With fb_query_sensors on (fb_rollout_sensor_read): sensordata [n][T][nsd], what fb_get(FB_SENSORDATA) returns
 *   after the step, and sensor_mean, what fb_get(FB_SENSOR_MEAN) returns (the same division by n_substeps).  The buffers are allocated
 *   on first use and grown when n T grows; -4 with a message when they do not fit.
 * Errors: no bank, n < 1 or n > n_envs, T < 1, n_substeps < 1, NULL ctrl, a slot out of range, never written or saved while its env
 * was held for a reset, a non-finite host input, applied-force sequences without the applied-force arrays, a feedback law of another
 * horizon.  fb_rollout synchronises; a device input is not checked.  fb_rollout_feedback: T >= 1 with both arrays, a tangent that does
 * not fit in shared memory, non-finite host values; it synchronises with host arrays.  The reads synchronise (any pointer may be NULL;
 * is_device: device pointers) and refuse before any rollout, or for sensors after a rollout with sensors off.  fb_rollout refuses a
 * call whose n differs from the law list's.                                                                                          */
int fb_rollout_feedback(FbHandle h, int T, const float* xref, const float* K, int is_device);
int fb_rollout_feedback_bank(FbHandle h, int L, int T, const float* xref, const float* K, const int32_t* law, int n, int is_device);
int fb_rollout(FbHandle h, const int32_t* slots, int n, int T, int n_substeps, const float* ctrl, const float* qfrc_applied,
               const float* xfrc_applied, int is_device);
int fb_rollout_read(FbHandle h, float* qpos, float* qvel, float* act, float* ctrl, float* time, int32_t* flags, int is_device);
int fb_rollout_sensor_read(FbHandle h, float* sensordata, float* sensor_mean, int is_device);
/* The iLQR backward pass (Tassa, Erez & Todorov 2012), batched over L problems of T steps, all in fp64 (nx = 2 nv + na, nu):
 *   inputs (host arrays, or device pointers when is_device): A [L][T][nx][nx] and B [L][T][nx][nu] (fp32, as fb_fd_read writes them),
 *   the cost gradients q [L][T+1][nx] and r [L][T][nu], the diagonal weights Q [nx], R [nu] and Qf [nx] shared by every problem, and
 *   the regularisation mu [L].  For t = T-1 .. 0 from s = q_T, P = diag(Qf):
 *     Qx = q_t + A's,  Qu = r_t + B's,  Qxx = diag(Q) + A'PA,  Quu = diag(R) + B'PB + mu I,  Qux = B'PA,
 *     k = -Quu^-1 Qu,  K = -Quu^-1 Qux  (Cholesky of Quu),  dV1 += k'Qu,  dV2 += k'Quu k / 2,
 *     s = Qx + K'Quu k + K'Qu + Qux'k,  P = sym(Qxx + K'Quu K + K'Qux + Qux'K).
 *   A Cholesky pivot that is not positive and finite sets status = t + 1 and stops that problem (its K, k and dV are then incomplete).
 * Five launches per step with no host synchronisation inside the pass; fixed-order sums and no atomics, so a problem's bits depend on
 * neither its index nor L.  The buffers are allocated on first use and grown with L T and L (a problem's workspace is
 * 8 (nx^2 + (nx + nu + 1)(2 nx + nu) + nu^2 + 2 nu (nx + 1)) bytes); -4 with a message when they do not fit.  Errors: L < 1, T < 1, a
 * NULL input, a model without actuators, nx + nu too large for the workspace's 32-bit offsets, a non-finite host input.  Weights of
 * any sign are accepted (an indefinite Quu reports its status).  It synchronises; a device input is not checked.
 * fb_lqr_read (synchronises; any pointer may be NULL; is_device: device pointers): K [L][T][nu][nx], k [L][T][nu], dV [L][2] (dV1, dV2)
 * and status [L] (int32); an error before any pass.                                                                                  */
int fb_lqr(FbHandle h, int L, int T, const float* A, const float* B, const double* q, const double* r, const double* Q, const double* R,
           const double* Qf, const double* mu, int is_device);
int fb_lqr_read(FbHandle h, double* K, double* k, double* dV, int32_t* status, int is_device);
/* Control-limited DDP (box-DDP; Tassa, Mansard & Todorov 2014): fb_lqr with bounds lower [L][T][nu] <= du_t <= upper [L][T][nu] on the
 * control change du = u - ubar of every problem step (fp64, +-inf allowed).  At each step k_t solves the box-constrained QP
 *   min 1/2 x'Quu x + Qu'x  subject to  lower_t <= x <= upper_t
 * by the projected Newton method of Tassa's boxQP, one warp per problem: from x = clamp(0), at most 100 iterations of
 *   g = Qu + Quu x; control i is clamped when x_i = lower_i and g_i > 0, or x_i = upper_i and g_i < 0; stop when every control is
 *   clamped; (re)factor the free block Quu_ff (Cholesky; on the first iteration and whenever the clamped set changed); stop when
 *   |g_free|_2 < 1e-8; dx_f = -Quu_ff^-1 g_f, dx_c = 0; a projected Armijo search from step 1: accept x_try = clamp(x + step dx) when
 *   (f(x_try) - f(x)) / (step dx'g) >= 0.1, else step *= 0.6, giving up below 1e-22; stop when the step lowers f by less than 1e-8 |f|.
 * Then the clamped set is taken again at the final x and its free block refactored if it changed.  K_t = -Quu_ff^-1 Qux_f on the free
 * rows and exactly 0 on the clamped ones; s, P and dV follow fb_lqr's formulas, which hold for any K and k.  A free block whose pivot is
 * not positive and finite sets status = t + 1, as fb_lqr's Cholesky.  Launches per step: fb_lqr's with the Cholesky and the solve
 * replaced by the QP and a masked solve; no host synchronisation inside the pass; fixed-order sums and no atomics, so a problem's bits
 * depend on neither its index nor L.  A problem's workspace grows by 8 4 nu + 4 nu bytes, a problem step's by 8 2 nu + 4 (nu + 2)
 * bytes (bounds, clamped set, QP record).  Errors: fb_lqr's, NULL bounds, and for host bounds a NaN, lower > upper, lower = +inf or
 * upper = -inf.  fb_lqr_read reads its K, k, dV and status.
 * fb_lqr_box_read (synchronises; any pointer may be NULL; is_device: device pointers): clamped [L][T][nu] (-1 at lower, +1 at upper,
 * 0 free, at the returned k) and qp [L][T][2] (accepted Newton steps, stop reason: -1 a free block that is not positive definite,
 * 0 no descent direction, 1 100 iterations, 2 the line search gave up, 4 a small improvement, 5 a small free gradient, 6 every control
 * clamped) (int32); an error before any pass and after a pass of fb_lqr.                                                            */
int fb_lqr_box(FbHandle h, int L, int T, const float* A, const float* B, const double* q, const double* r, const double* Q,
               const double* R, const double* Qf, const double* mu, const double* lower, const double* upper, int is_device);
int fb_lqr_box_read(FbHandle h, int32_t* clamped, int32_t* qp, int is_device);
/* Sampling-based MPC: MPPI (Williams et al. 2017, the information-theoretic update without the control cross term, R pricing the
 * controls) and predictive sampling (Howell et al. 2022, MuJoCo MPC), batched over L tracking problems of K = n_samples samples each
 * (nx = 2 nv + na, nr = nq + nv + na).  Problem l starts from state-bank row slots[l] with the nominal control sequence mean[l] [T][nu].
 * One iteration:
 *   sample:   sample k of problem l is u_k,t = clamp(mean_t + sigma * eps_k,floor(t / hold)), the clamp on ctrl-limited actuators only
 *             (what the actuation stage applies), eps a standard normal (Box-Muller in fp64) of a counter hash of (seeds[l], iteration,
 *             k, knot, actuator): the noise of a problem depends on its seed alone, never on its index or L.  Sample 0 has eps = 0
 *             (the clamped mean).  hold >= 1 is the zero-order-hold knot spacing in control steps.
 *   roll out: all L K samples open loop, T control steps of n_substeps substeps, sample (l, k) in env l K + k from row slots[l] (its
 *             parameter overlay and applied forces included, as fb_rollout); envs past L K run copies of the last sample.  The step
 *             kernels, the rollout input kernel and the step graph run as fb_rollout runs them.
 *   score:    J_k = 1/2 sum_{t<T} (|x_t (-) xref_t|^2_Q + |u_k,t - uref_t|^2_R) + 1/2 |x_T (-) xref_T|^2_Qf, (-) fb_fd_transition's
 *             tangent, summed in fp64 from the fp32 state, the lane partials in lane order.  A sample whose env sets the bad-state
 *             flag (flag bit value 1: |qacc|^2 >= 1e28, or a non-finite qacc or qvel) scores +inf, and so does a NaN cost.
 *   update:   temperature > 0 (MPPI): w_k = exp(-(J_k - J_min) / temperature) (+inf: 0), mean_t = sum_k w_k u_k,t / sum_k w_k in fp64,
 *             stored fp32.  temperature = 0 (predictive sampling): mean = the lowest-cost sample, bit for bit (ties: the lowest k).
 *             If every sample scores +inf the mean stays and status = 1 + the iteration (the first such).
 * One warp per work unit (a sample, a problem, or a problem's block of steps), no atomics and no shared memory: every sum has a fixed
 * order, so a problem's bits depend on neither its index, nor L, nor the other problems.
 * fb_plan_program sets the program for the calls that follow: n_samples >= 2, hold >= 1, temperature >= 0 and finite, sigma [nu] (fp32),
 * Q [nx], R [nu], Qf [nx] (fp64 diagonal weights) >= 0 and finite, read when the call is made.  NULL or n_samples = 0 clears it.  Errors
 * also: a model without actuators.  It synchronises.
 * fb_plan copies its inputs and the fan-out list once, then runs n_iter iterations with no host copy or synchronisation: inputs
 * (host rows, or device pointers when is_device) mean [L][T][nu], xref [L][T + 1][nr] and uref [L][T][nu] (NULL: 0); slots [L] and
 * seeds [L] are host arrays.  Its buffers are its own,
 * allocated on first use and grown with L n_samples T, L (T + 1) and L n_iter; -4 with a message when they do not fit.  It does not
 * touch fb_rollout_read's records, the feedback law or the bank; afterwards the envs are a workspace.  Errors: no bank, no program,
 * L < 1 or L n_samples > n_envs, T < 1, n_substeps < 1, n_iter < 1, a NULL input, a slot out of range, never written or saved while
 * its env was held for a reset, a non-finite host input.  It synchronises; a device input is not checked.
 * fb_plan_read (synchronises; any pointer may be NULL; is_device: device pointers): mean [L][T][nu] after the last update, cost
 * [L][n_iter][2] (per iteration: the nominal's cost, i.e. sample 0's, and the lowest cost), sample_cost [L][n_samples] and samples
 * [L][n_samples][T][nu] of the last iteration, status [L] (int32); an error before any plan.                                        */
typedef struct FbPlanProgram {
  int32_t n_samples;                           /* K >= 2 samples per problem (0: clear)                                      */
  int32_t hold;                                /* control steps per noise knot, >= 1                                           */
  double temperature;                          /* > 0: MPPI; 0: predictive sampling                                           */
  const float* sigma;                          /* [nu] noise scale per actuator                                               */
  const double *Q, *R, *Qf;                    /* [nx], [nu], [nx] diagonal weights                                           */
} FbPlanProgram;
int fb_plan_program(FbHandle h, const FbPlanProgram* p);
int fb_plan(FbHandle h, const int32_t* slots, int L, int T, int n_substeps, int n_iter, const uint32_t* seeds, const float* mean,
            const float* xref, const float* uref, int is_device);
int fb_plan_read(FbHandle h, float* mean, double* cost, double* sample_cost, float* samples, int32_t* status, int is_device);
/* ---- system identification: the normal equations of parameter fits (fb_sid.h; flybody_b200.sysid is the front end) -------------
 * fb_sid_accumulate adds the weighted normal equations of L fit problems from the outputs the last parameter-Jacobian query left on the
 * device; nothing of the Jacobians is read back.  query FB_SID_TRANSITION reads the last fb_fd_param_transition: FD problem i's residual
 * r = x'_pred (-) x'_obs [nx], x'_pred the nominal next state (fb_fd_param_read's), (-) fb_fd_transition's tangent
 * (mj_differentiatePos(x'_obs qpos, x'_pred qpos), then the qvel and act differences), J = dxdp [nx][k].  FB_SID_INVERSE reads the last
 * fb_fd_param_inverse: r = qfrc_inverse - target [nv], J = DfDp^T.  Per fit problem l, over the FD problems i with problem[i] = l, in
 * fp64 from the fp32 outputs:
 *   H_l += c_i J^T W J,  g_l += c_i J^T W r,  cost_l += c_i r^T W r / 2,  count_l += 1
 * W = diag(weight), c_i = sample_weight[i]; a transition with c_i = 0 adds nothing (as problem[i] = -1).  A transition whose residual or
 * Jacobian is not finite, or (transition) whose nominal env set the bad-state flag (bit value 1), adds +inf to cost_l and 1 to bad_l and
 * nothing to H_l or g_l.  No atomics: each transition's term is one fixed-order sum, added in transition order, so a problem's bits
 * depend on neither its index, nor L, nor the other problems, nor on how its transitions are split across calls.
 * Inputs: problem [n] (host int32, a fit problem in [0, L) or -1: skip), target (x'_obs [n][nq + nv + na] of a transition, the qfrc target
 * [n][nv] of an inverse, NULL: 0), sample_weight [n] (fp32 >= 0, NULL: 1), target and sample_weight host rows or device pointers when
 * is_device; weight [nx] or [nv] (host fp64 >= 0 and finite).  reset = 1 starts the L problems' sums from 0; reset = 0 adds to them.
 * Its buffers are its own, allocated on first use and grown with n, L (k^2 + k + 1) and L; -4 with a message when they do not fit.
 * Errors: an unknown query, no result of that query, any kernel launched on the handle since it (fb_launch_count: the outputs and the
 * nominal envs' flags must be the query's own), n other than the query's, L < 1, L or k other than the sums' without reset (or no sums),
 * a problem id out of range, a NULL problem or weight, a NULL transition target, negative or non-finite host weights, a non-finite host
 * target.  It synchronises; a device input is not checked.
 * fb_sid_read (synchronises; any pointer may be NULL; is_device: device pointers): H [L][k][k] (symmetric), g [L][k], cost [L], count
 * [L] and bad [L] (int32) of the sums; an error before any fb_sid_accumulate.                                                         */
enum FbSidQuery { FB_SID_TRANSITION = 0, FB_SID_INVERSE = 1 };
int fb_sid_accumulate(FbHandle h, int query, int L, const int32_t* problem, int n, const float* target, const double* weight,
                      const float* sample_weight, int reset, int is_device);
int fb_sid_read(FbHandle h, double* H, double* g, double* cost, int32_t* count, int32_t* bad, int is_device);
int fb_n_envs(FbHandle h);
int fb_n_envs_padded(FbHandle h);
void* fb_stream(FbHandle h);                 /* cudaStream_t the handle launches on */
int fb_sync(FbHandle h);
long long fb_launch_count(FbHandle h);       /* kernels launched by this handle so far */
/* device time (ms) of the last fb_step measured with CUDA events on the handle's stream */
float fb_last_step_ms(FbHandle h);
/* solver configuration: tolerance and iteration cap of the constraint solver */
/* per-kernel device timing (CUDA events around every launch while enabled): cumulative ms and launch
 * counts per pipeline stage; fb_profile_name(kind) names the stage.  Used by bench.py's roofline block. */
int fb_profile(FbHandle h, int enable);
int fb_profile_read(FbHandle h, double* ms, long long* counts, int n);
const char* fb_profile_name(int kind);
/* Shared-memory budget of the seven step kernels (kinds smooth, solve, finish, pos, col, proj, vel of fb_profile_name): the
 * dynamic shared memory one CTA of 4 warps requests when this handle launches it, and the CTAs of that kernel that fit on one
 * SM of the handle's device at that size (cudaOccupancyMaxActiveBlocksPerMultiprocessor; 0 in a build without a device).
 * The kernels are compiled for 8 resident CTAs per SM, which puts 4096 envs in one wave on an H100.
 * Returns -1 for a kind that is not a step kernel.                                                                      */
int fb_step_kernel_smem(FbHandle h, int kind, int* bytes_per_cta, int* blocks_per_sm);
int fb_set_solver(FbHandle h, float tolerance, int max_iter);
const char* fb_last_error(FbHandle h);
const char* fb_version(void);

#ifdef __cplusplus
}
#endif
#endif
