// fb_types.h -- device-side model / state layout of the batched fly stepper.
//
// Thread mapping / layout rule (DESIGN.md "Data layout in HBM"): ONE WARP OWNS ONE ENVIRONMENT.  The 32
// lanes of the warp split the env's intra-step parallelism (branch lists of the kinematic tree, pair
// chunks of the collision list, constraint rows, dofs); synchronisation is __syncwarp only and every env
// runs its own data-dependent trip counts.  All per-env state and intermediates live in one fp32/int32
// RECORD per env (array-of-records, `rec` 4-byte slots apart), so the lanes of a warp touch neighbouring
// addresses of the same record.  Model constants are small read-only arrays read through the constant
// bank / L1.
#pragma once
#include <stdint.h>
#include "../../include/flybody_b200.h"

#ifdef __CUDACC__
#define FB_DEV __device__ __forceinline__
#define FB_DEVN __device__ __noinline__
#define FB_HD __host__ __device__
#define FB_DEVM __device__ __forceinline__   // a member function of a kernel's parameter
#else
#define FB_DEV static inline
#define FB_DEVN static
#define FB_HD
#define FB_DEVM
#endif

#define FB_NY 32             // lanes per env (threadIdx.x); every kernel runs 32 lanes per env
#define FB_MINB 8            // resident blocks per SM the kernels are compiled for: 8 x 4 warps >= 4096 envs / 132 SMs (H100), one wave
#define FB_WPB 4             // envs (warps) per block
#define FB_NLMAX 10          // branch lists of the tree kernels (lanes 0..nlist-1 active; 3 lanes per list in the factorisation)
#define FB_ROWPAR 8          // rows processed in parallel by the projection kernel
#define FB_MINVAL 1e-15f

// Warp-cooperative code is written as WPAR sections: on the GPU every lane runs the section body and the
// section ends in a warp barrier; the host emulation (tests only) runs the 32 lanes one after the other.
// Code between sections is warp-uniform.
#ifdef __CUDACC__
#define WPAR_BEGIN { const int lane = threadIdx.x; (void)lane;
#define WPAR_END } __syncwarp();
#define FB_WARPFN __device__ __forceinline__
#else
#define WPAR_BEGIN for (int lane = 0; lane < 32; lane++) {
#define WPAR_END }
#define FB_WARPFN static inline
#endif
// Lane registers of warp functions: a register per lane on the GPU, an array over the 32 lanes in the host emulation
// (where a WPAR section runs lane after lane: a value read through SHF / BALLOT must have been written in an EARLIER section).
#ifdef __CUDACC__
#define LREG(type, name) type name
#define L(name) name
#define SHF(name, src) __shfl_sync(0xffffffffu, name, (src) & 31)
#define LREGA(type, name, K) type name[K]             /* K registers per lane: every index must be a compile-time constant after unrolling */
#define LA(name, k) name[k]
#define SHFA(name, k, src) __shfl_sync(0xffffffffu, name[k], (src) & 31)
#define BALLOT(out, name, cmp) out = __ballot_sync(0xffffffffu, (name)cmp)
#define POPC(x) __popc(x)
#define FFS(x) __ffs((int)(x))
#else
#define LREG(type, name) type name[32] = {}
#define L(name) name[lane]
#define SHF(name, src) name[(src) & 31]
#define LREGA(type, name, K) type name[K][32] = {}
#define LA(name, k) name[k][lane]
#define SHFA(name, k, src) name[k][(src) & 31]
#define BALLOT(out, name, cmp) { out = 0; for (int l_ = 0; l_ < 32; l_++) if ((name[l_])cmp) out |= 1u << l_; }
#define POPC(x) __builtin_popcount(x)
#define FFS(x) __builtin_ffs((int)(x))
#endif


struct alignas(8) FsItem { unsigned x, y; };
struct DevModel {
  // sizes / options
  int nq, nv, nu, na, nbody, njnt, ngeom, npair, nsite, ntendon, nwrap, nsensor, nsensordata, nM, nfluid;
  int noslip_iterations, cone_elliptic, max_iter, ls_iter, solve_ncap; float solve_rtol;
  float timestep, gravity[3], density, viscosity, wind[3], impratio, tolerance, noslip_tolerance, meaninertia, ls_tolerance;
  // tree partition
  int nroot, nlist;
  const int *root_body;                    // [nroot]
  const int *list_adr, *list_num, *list_body, *list_root;   // bodies of each branch list in topological order
  int max_list_ndof;                       // dofs of the longest list (steps of the lock-step sweeps)
  // bodies
  const int *body_parentid, *body_jntadr, *body_jntnum, *body_dofadr, *body_dofnum, *body_lastdof,
      *body_fluid_ellipsoid, *body_isroot, *body_sensacc, *body_sensfrc;
  const float *body_pos, *body_quat, *body_ipos, *body_iquat, *body_mass, *body_inertia, *body_invweight0;
  // joints / dofs
  const int *jnt_type, *jnt_qposadr, *jnt_dofadr, *jnt_bodyid, *jnt_limited;
  const float *jnt_pos, *jnt_axis, *jnt_stiffness, *jnt_range, *jnt_solref, *jnt_solimp, *jnt_margin, *qpos0, *qpos_spring;
  const int *dof_bodyid, *dof_jntid, *dof_parentid, *dof_Madr, *dof_subend, *dof_depth /* #non-root ancestors; local index for root dofs */, *dof_chainlen, *dof_anc /* [nM] t-th ancestor of the row's dof */;
  const unsigned char* dof_lca;   // [nv][nv] number of common ancestors-or-self of two dofs (= chain length of their lowest common ancestor, 0: none)
  const int *dof_rootidx /* root (index into root_body) a list dof hangs off, -1 for root dofs */, *root_haslists;
  const unsigned* tsolve_blob; int ts_hdr_words, ts_nm_pad, ts_blob_words;    // sweep program copied per CTA into shared memory (fb_tree.h)
  const unsigned* fs_rng; const FsItem* fs_items;   // factorisation schedule: per (step, lane) first item | count << 16; item = (adr_k | t << 12 | update length << 18, adr of the ancestor row)
  const float* M_damp;         // per entry of the packed inertia: joint damping on the diagonals, 0 elsewhere
  const int* body_adhesion;    // adhesion actuator acting on the body, or -1
  const float *dof_armature, *dof_damping, *dof_invweight0;
  // geoms
  const int *geom_type, *geom_bodyid, *geom_condim;
  const float *geom_size, *geom_pos, *geom_quat, *geom_rbound, *geom_friction, *geom_solmix, *geom_solref, *geom_solimp,
      *geom_margin, *geom_gap;
  const int *pair_geom1, *pair_geom2;
  const int* pair_info; const float* pair_rsum;   // packed broadphase record: g1 | g2 << 15 | plane << 30, margin + bounding radii
  // fluid geoms, sites, tendons, actuators, sensors
  const int *fluid_bodyid; const float *fluid_pos, *fluid_quat, *fluid_size, *fluid_coef;
  const int *site_bodyid, *site_type; const float *site_pos, *site_quat, *site_size;
  const int *tendon_adr, *tendon_num, *wrap_dofid, *wrap_qposadr; const float *wrap_coef;
  const int *actuator_trntype, *actuator_trnid, *actuator_dyntype, *actuator_biastype, *actuator_ctrllimited,
      *actuator_forcelimited, *actuator_actadr;
  const float *actuator_dynprm, *actuator_gainprm, *actuator_biasprm, *actuator_ctrlrange, *actuator_forcerange;
  const int *sensor_type, *sensor_objid, *sensor_adr, *sensor_dim;
};

// efc row types
enum { FB_CT_LIMIT = 0, FB_CT_FRICTIONLESS = 1, FB_CT_ELLIPTIC = 2 };

struct DevTask;
struct DevData {
  int N, Np;                   // envs, padded envs
  unsigned rec;                // record stride (4-byte slots) between consecutive envs
  int nsub_done, sens_mode, do_integrate;
  // integrated state
  float *qpos, *qvel, *act, *ctrl, *qacc, *dof_isd /* D^-1/2 of the current factor */, *time;
  // position stage
  float *ref;                  // [3] reference point (root position) all spatial quantities are taken about
  float *xpos, *xquat, *xmat, *xipos, *ximat;          // body frames (positions relative to ref)
  float *geom_xpos, *geom_xmat, *site_xpos, *site_xmat;
  float *Sang, *Slin;          // [nv*3] motion subspaces about ref
  float *inert10, *crb10;      // [nbody*10]
  float *qM, *qLD, *qLDe;      // [nM] inertia, its L^T D L factor, factor of M + h*diag(damping)
  // velocity stage
  float *bvel, *bacc, *bfrc, *bfl, *bfrc0, *bdel;   // [nbody*6] spatial velocity, bias accel, bias force (subtree sums), fluid wrench, per-body bias force
  float *qfrc_bias, *qfrc_passive, *qfrc_actuator, *qfrc_smooth, *qfrc_zf /* Z^T f */, *qfrc_constraint, *qtmp /* D^-1 L^-T qfrc_smooth */;
  float *act_dot, *actuator_force;
  // contacts
  int *ncon; float *con_dist, *con_pos, *con_frame; int *con_geom1, *con_geom2, *con_efcadr, *con_dim;
  float *con_mu, *con_fric;    // mu, friction[2]
  float *tmp_con; int *tmp_geom;   // collision candidates' contacts, before compaction
  // constraints
  int *nefc; int *efc_type, *efc_id;
  float *efc_pos, *efc_margin, *efc_D, *efc_R, *efc_K, *efc_B, *efc_imp, *efc_aref, *efc_b, *efc_force;
  float *efc_J, *efc_Z;        // [MAXEFC][FB_JROW] chain-sparse rows (fb_constraint.h: EJC)
  float *efc_A, *efc_G;        // packed lower triangles
  int *efc_key, *prev_key, *prev_n; float *prev_lam;   // warm start: constraint forces of the previous solve, matched by row identity
  float *efc_w;                // [8*MAXEFC] solver work vectors
  int *efc_la, *efc_lb;       // row dof chains
  // sensors / outputs
  float *sensordata, *sensor_sum;
  int clk_launch; long long* clk;              // -DFB_CLK builds only: clock64() of warp 0 after every stage of every launch (latency profile)
  int *flags, *niter, *hold;   // hold != 0: env is not integrated by the next fb_step (pending reset)
  const int* rst_ids; const float* rst_qpos; const float* rst_qvel; int rst_n, rst_has_qvel, rst_hold;   // staged partial reset
  float* sc_field; const int* sc_idx; const float* sc_vals; int sc_k, sc_nan0;                                 // staged column scatter
  unsigned sc_stride;          // slots between the scatter target's env rows: 0 = a record field, else a compact [Np][sc_stride] array
  float *obs;                  // packed AoS observation [N][obs_dim]
  int obs_dim;
  // task observation program (fb_obs_program): final observation rows [N][tobs_dim]
  float *tobs; int tobs_dim, op_n, op_root_body, op_ref_len, op_nsub, op_ref_slot /* 1: op_ref is [N][op_ref_len][7], one table per env */;
  const int *op_kind, *op_a, *op_b, *op_off, *op_list; const float* op_ref; const int* op_step; const unsigned char* op_first;
  const struct DevTask* task;  // device-side task logic, or nullptr
  // applied forces (mjData.qfrc_applied, mjData.xfrc_applied): compact [Np][nv] and [Np][nbody][6] (world force, then torque, at the
  // body's CoM), allocated together on first use (fb_applied_ptrs / fb_set / fb_write_state); nullptr until then and after
  // fb_clear_applied, so a step that never set them runs without the term
  float *qfrc_applied, *xfrc_applied;
  // model-parameter overlay (fb_param_*): compact [Np][prm_stride], parameter p (enum FbParam) of an env at prm_off[p] of its row,
  // body_inertia padded to four floats per body as the model table; nullptr until first use and after fb_param_clear, so a step that
  // never set parameters reads the compiled tables.  prm_mdamp: the row's derived M_damp [nM] (DevModel::M_damp of the env's dof_damping).
  // prm_count: the env's draws so far; prm_draw: the draw program of resets, or nullptr
  float* prm; unsigned prm_stride; int prm_off[FB_NPARAMS], prm_mdamp; unsigned* prm_count; const struct DevPrmDraw* prm_draw;
};
// draw program of the overlay (fb_param_draws): parameter p with on[p] takes lo + u (hi - lo) at each reset, u one draw per element
// (or one for all of them: shared[p]); n[p] values per env; lo, hi are laid out as an overlay row
struct DevPrmDraw {
  unsigned seed; int on[FB_NPARAMS], shared[FB_NPARAMS], n[FB_NPARAMS];
  const float *lo, *hi;
};

// Device-side task logic (fb_task_program): what the reference's task hooks do around the physics step -- auto-reset,
// ghost placement, wing-beat pattern generator, termination, reward, discount -- for the shared-reference (inference)
// form of walk_imitation / flight_imitation, and for both with a trajectory dataset (ref_bank).  Lives in device memory;
// DevData::task points at it.
#define FB_RBANK_W 15                      // flight bank row: root qpos 7, CoM qvel 6, CoM x, y 2 (the first 15 columns of every bank row)
struct DevTask {
  int kind;                                // enum FbTaskKind (include/flybody_b200.h)
  int root_qadr, root_vadr, ghost_qadr, ghost_vadr, root_body, user_col /* action column of the beat-frequency action, -1: none */;
  float ghost_offset[3], dt, time_limit, term_com, term_linvel, term_angvel, term_qacc, term_height;
  int velocimeter_adr, gyro_adr, com_body, ref_len, obs_refdisp_off, obs_refquat_off;
  const float *reset_qpos, *ref_qpos /*[ref_len][7]*/, *ref_qvel /*[ref_len][6]*/;
  int n_noise; const int* noise_qadr; float noise_amp; unsigned seed;
  int n_wing; const int *wing_qadr, *wing_vadr, *wing_ctrl;
  int n_freq, tab_len; const float *wb_traj /*[n_freq][tab_len][n_wing]*/, *wb_phase, *wb_phase_mod /*[n_freq][tab_len], +inf padded*/, *wb_freqs; const int* wb_len;
  float wb_base_freq, wb_rel_range, wb_rate, com_offset[3];
  // FB_TASK_VISION (vision_guided_flight): ranges of the per-episode draws, hover pose, terrain bank and the env's own heightfield buffers
  float th_rng[2], ts_rng[2], x_rng[2], y_rng[2], hover_quat[4], target_zaxis[3]; int fatal;
  int n_bank, hf_nrow, hf_ncol, hf_ncm; float hf_half;
  const float *bank, *bank_hmax, *bank_cmax; float *hf_data, *hf_hmax, *hf_cmax;
  float* target;                           // [N][2] target height, target speed of the running episode
  int trench_cap; const float *trench_x, *trench_y; const int* trench_len; int* pick;   // 'trench' arenas: centre line per bank terrain; the env's terrain
  // FB_TASK_WALK / FB_TASK_FLIGHT with ref_bank (dataset): trajectory bank [rows][rbank_w] (fb_ref_bank / fb_ref_bank_wide), picks, the env's reference slot
  int ref_bank, n_pick, randomize_start, start_margin, max_episode_rows, future_steps, slot_len, rbank_w;
  const float* rbank; const int *traj_off, *traj_len, *pick_traj; float* slots /* [N][slot_len][7] */;
  int *ep_traj, *ep_start, *ep_row0, *ep_n;   // the running episode: trajectory, start step, bank row of its row 0, rows in use
  int* pin;                                // [N][3] has pin, trajectory, start step of the next reset (fb_task_ref_pick)
  // FB_TASK_WALK with ref_bank (walking dataset): the dataset's joints / sites, the observation columns of the walker features, the DeepMimic
  // reward's constants; bank row after the 15 root columns: mocap qpos [nj], mocap qvel [nj], root2site [ns][3], joint_quat [nj][4]
  int n_mjnt, n_msite; const int* mocap_qadr; const float* wing_spring;
  int obs_root_pose_off, obs_root_qvel_off, obs_mocap_qpos_off, obs_mocap_qvel_off, obs_mocap_axes_off, obs_mocap_sites_off, obs_wing_qpos_off;
  float dm_std[4], dm_weight[4], retract_margin;
  float* rw_part;                          // [N][FB_NY][3] per-lane partial sums of the joint / site terms of the reward (ktask_reward)
  // per-env state
  int *step, *needs_reset, *resetting, *episode, *ep_steps /* step index that ends the episode */, *wb_idx, *wb_pos, *has_uniform;
  float *uniform /* [N][8] */, *wb_freq;
  int* op_step; unsigned char* op_first;   // the observation program's per-env inputs, maintained here instead of by fb_task_inputs
  float* out;                              // [N][4] reward, discount, step_type (0 FIRST, 1 MID, 2 LAST), 0
  // FB_TASK_BALL (walk_on_ball): the ball joint's first dof, the target ball velocity and the reward's margin
  int ball_vadr; float ball_target[3], ball_margin;
};

// A compiler barrier at both ends of a branch that only some models take (ball joints).  Without it the optimiser may hoist
// or sink arithmetic that branch shares with its neighbours (free and hinge joints) across the branch, so that a multiply and its add
// end up in different blocks and are no longer fused: the other models' results would change in the last bits.
#define FB_NO_MERGE() asm volatile("" ::: "memory")
#ifdef __CUDACC__
#define FB_FLAG_OR(bit) atomicOr(&AT(d.flags, 0), (bit))
#else
#define FB_FLAG_OR(bit) (AT(d.flags, 0) |= (bit))
#endif
