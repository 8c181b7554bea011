// flybody_b200.cu -- C ABI (include/flybody_b200.h) + kernel launch sequence of the batched fly
// stepper for sm_90a (H100).
//
// One control step = n_substeps x [ step2 ; step1 ] exactly as dm_control's legacy Physics.step()
// (SURVEY.md App. A), each substep being the staged kernel pipeline
//   step2: k_act -> k_smooth(solve) -> k_ref -> k_solve -> k_finish(qacc, sensors, Euler)
//   step1: k_pos(kinematics, CRB, factor) -> k_col -> k_con -> k_proj(J, Z, A) -> k_vel(RNE, passive)
// One warp per env, all per-env data in one record per env (fb_types.h).
//
// The same translation unit compiles as plain C++ with -DFB_EMU (tests/_emu): phases run in
// nested host loops.  That build exists ONLY so CPU tests can exercise the kernel source; the
// Python package never loads it (flybody_b200/stepper.py refuses to run without the CUDA library).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <algorithm>
#include <cmath>
#include <limits>

#ifndef FB_EMU
#include <cuda_runtime.h>
#endif
#include "fb_solver_reg.h"
#include "fb_render.h"
#include "fb_hfield.h"
#include "fb_task.h"
#include "fb_state.h"
#include "fb_ik.h"
#include "fb_inverse.h"
#include "fb_fd.h"
#include "fb_rollout.h"
#include "fb_lqr.h"
#include "fb_plan.h"
#include "fb_sid.h"

enum { K_ACT = 0, K_SMOOTH, K_REF, K_SOLVE, K_FINISH, K_POS, K_COL, K_CON, K_PROJ, K_VEL, K_SENS, K_PACK, K_MISC, K_NKIND };
static const char* const kKindNames[K_NKIND] = {"act", "smooth", "ref", "solve", "finish", "pos", "col", "con", "proj", "vel", "sens", "pack", "misc"};
// one finite-difference query (fb_fd.h): what it is, and its last call
struct FdQuery {
  const char *name, *cols, *what;         // the compute entry, its columns entry, what a read before any call finds missing
  bool inverse, param;                    // evaluation: the inverse dynamics (else the step); inputs: parameter directions (else the state)
  DevFdQ p = {};                          // the last call's kernel parameter; the blocks' and nominals' out are the query's outputs
  std::vector<void*> scope, sens_scope;   // the outputs and the sensor outputs, allocated on the first call (with sensors on)
  int done = 0; bool sens = false;        // problems of the last call; it ran with sensors on
  long long at = 0;                       // fb_launch_count when the last call returned (fb_sid_accumulate reads its outputs and flags)
};
// the scratch the queries share, no read returns it; each part is allocated on the first call that needs it
struct FdScratch {
  float* delta;                           // [Np]
  DevInv inv; float *qpos, *qvel, *qacc;  // the inverses': every env's DevInv; the problems [N/2][nq], [N/2][nv], [N/2][nv]
  float* rows;                            // [N/2][prm_stride] the parameter inverse's overlay rows
  float* sens;                            // [Np][nsd] every env's sensors (of x for a transition, kinv_sensors' for an inverse)
};
struct Pool { std::vector<void*> bufs; size_t cap = 0; };   // buffers for `cap` rows, replaced as a whole when a call needs more (grow)
// Every device buffer allocated after fb_create belongs to one scope (a list of buffers, or a Pool's): it is freed after a stream sync
// when its scope is replaced or grown, and by fb_destroy.
struct FbSim {
  DevModel m; DevData d;
  int prof_on; double prof_ms[K_NKIND]; long long prof_n[K_NKIND];
  FbModel hm;                       // host copy of scalar fields (pointers invalid after create)
  std::vector<void*> allocs;
  std::vector<void*> obs_scope, task_scope;   // device buffers of the current observation / task program: freed when the program is replaced
  std::vector<void*> applied_scope;           // qfrc_applied / xfrc_applied: freed by fb_clear_applied
  std::vector<void*> prm_scope;               // parameter overlay, draw counters and draw program (fb_param_*): freed by fb_param_clear
  std::vector<float> h_prm0; int prm_n[FB_NPARAMS];   // the overlay row of the compiled model; values per env of each parameter
  DevPrmDraw prm_draw_host; DevPrmDraw* prm_draw_dev; std::vector<float> h_prm_lo, h_prm_hi;   // the draw program and its ranges (row layout)
  std::vector<void*> ref_scope, bank_scope;   // reference slots (fb_ref_slots) / terrain bank (fb_hfield_bank): freed when replaced
  std::vector<int> h_dof_parent, h_dof_Madr, h_body_parent;
  std::vector<int> h_jnt_type, h_jnt_qadr, h_jnt_dofadr, h_jnt_body, h_site_body;   // joint / site tables an IK program is checked and built against
  std::vector<double> h_qpos0;
  DevIk ik = {}; std::vector<void*> ik_scope; int ik_solved = 0;   // inverse kinematics (fb_ik_program): parameters and buffers; problems of the last solve
  DevInv inv = {}; std::vector<void*> inv_scope; int inv_done = 0;   // inverse dynamics (fb_inverse): buffers, allocated on first use; problems of the last call
  // sensor outputs of the dynamics queries (fb_query_sensors): buffers allocated on the first call with sensors on; inv_sens: the last
  // fb_inverse ran with sensors on
  int sens_on = 0;
  float* inv_sd = nullptr; std::vector<void*> inv_sd_scope; bool inv_sens = false;              // fb_inverse: sensordata [Np][nsd]
  // finite-difference Jacobians (fb_fd_*; fb_fd.h): the four queries, the scratch they share, and the parameter direction program
  // (k directions, any scale among them) with its device tables
  FdQuery fd_tr{"fb_fd_transition", "fb_fd_columns", "transition", false, false};
  FdQuery fd_inv{"fb_fd_inverse", "fb_fd_inverse_columns", "Jacobians", true, false};
  FdQuery fd_ptr{"fb_fd_param_transition", "fb_fd_param_columns", "parameter Jacobians", false, true};
  FdQuery fd_pinv{"fb_fd_param_inverse", "fb_fd_param_columns", "parameter Jacobians", true, true};
  FdScratch fdx = {};
  DevFdPrmProg fdp_prog = {}; std::vector<void*> fdp_prog_scope; int fdp_k = 0; bool fdp_scale = false;
  // rollouts (fb_rollout*; fb_rollout.h): inputs and records of n T rows, grown on demand in three pools (ctrl and the records;
  // applied-force inputs; sensor records); the feedback bank of roll_fb_L laws of roll_fb_T steps (fb_rollout_feedback_bank) in a pool
  // of L T law steps, and its law list of roll_fb_n rollouts (0: every rollout takes law 0); rows of the last call
  DevRoll roll = {}; Pool roll_pool, roll_app_pool, roll_sd_pool;
  float *roll_xref = nullptr, *roll_K = nullptr; int* roll_law = nullptr; Pool roll_fb_pool, roll_law_pool; int roll_fb_T = 0, roll_fb_L = 0, roll_fb_n = 0;
  float *roll_qf = nullptr, *roll_xf = nullptr, *roll_sd = nullptr, *roll_sm = nullptr;   // applied-force inputs, sensor records
  int roll_done = 0; bool roll_sens = false;
  // the iLQR backward pass (fb_lqr; fb_lqr.h): inputs and outputs of L (T + 1) problem steps and the workspace of L problems, grown on
  // demand; problems and steps of the last call
  DevLqr lqr = {}; Pool lqr_pool, lqr_ws_pool; int lqr_done = 0;
  // its box-constrained form (fb_lqr_box): bounds and QP records of L T problem steps, the QP workspace of L problems; lqr_box: the last
  // pass had bounds
  DevLqrBox lqr_b = {}; Pool lqr_box_pool, lqr_qp_pool; bool lqr_box = false;
  // sampling-based MPC (fb_plan_program / fb_plan; fb_plan.h): the program (plan.K > 0: set) and its weights; the buffers, grown on demand
  // with L K T (the samples), L K (their costs and weights), L (T + 1) (mean, xref, uref and the per-problem words) and L n_iter (the
  // record); the rollout parameter of the samples; problems of the last call
  DevPlan plan = {}; DevRoll plan_roll = {}; std::vector<void*> plan_prog_scope; Pool plan_s_pool, plan_k_pool, plan_l_pool, plan_h_pool; int plan_done = 0;
  // system identification (fb_sid_accumulate / fb_sid_read; fb_sid.h): the transition scratch (grown with n), the sums of sid_L problems
  // of sid_k directions (grown with L (k^2 + k + 1); sid_L = 0: none yet) and the per-problem words (grown with L + 1)
  DevSid sid = {}; Pool sid_t_pool, sid_s_pool, sid_l_pool;
  int sid_L = 0, sid_k = 0;
  int device; long long launches; float last_ms; std::string err;
  int first_substep = 1; int hold_pending;
  int* rst_ids_dev; float* rst_qpos_dev; float* rst_qvel_dev; Pool rst_pool;   // reset lists (do_reset)
  const int* act_map_dev; int n_action; std::vector<void*> act_map_scope;
  int blob_in_smem;            // copy the sweep program of the triangular solves into shared memory per CTA (default: for batches <= 1024 envs; FB_BLOB=0/1 overrides)
  int* op_step_dev; unsigned char* op_first_dev;
  float* ref_slots; int ref_slot_len;      // per-env reference tables (fb_ref_slots)
  float* rbank_dev; int *rbank_off_dev, *rbank_len_dev, rbank_w; std::vector<int> rbank_len; std::vector<void*> rbank_scope;   // trajectory bank (fb_ref_bank_wide)
  DevHf hf; bool hf_on; int hf_nrow, hf_ncol; std::vector<void*> hf_pair_scope;      // heightfield collision (fb_hfield_collision)
  float *bank_dev, *bank_hmax_dev, *bank_cmax_dev; int bank_n;      // terrain bank of the device-side vision task (fb_hfield_bank)
  float* hfield_dev; float* hmax_dev; float* cmax_dev; int hf_nbr, hf_nbc; std::vector<void*> hf_scope;   // per-env heightfields (ensure_hfield)
  DevEye eye; unsigned char* eye_out; size_t eye_bytes; std::vector<void*> eye_scope;                 // eye cameras (fb_eye_program)
  DevTask task_host;                       // host copy of the device-side task program (its pointers are device pointers)
  float* stage; int* stage_i; Pool stage_pool, stage_i_pool; unsigned ws_slot;   // staging buffers (ensure_stage)
  // state bank (fb_state_*): [st_slots][st_row] rows of the layout in st_segs; dropped (st_stale) when a program that shapes the layout is replaced
  unsigned* st_bank = nullptr; int st_slots = 0; unsigned st_row = 0; bool st_stale = false; uint64_t st_sig = 0;
  StSeg* st_segs_dev = nullptr; int st_nseg = 0, st_hold_off = 0; std::vector<void*> st_scope;
  std::vector<char> st_written;            // per slot: 0 never written, 1 written, 2 written while an env may be held for its reset
  int* st_ids_dev = nullptr; Pool st_ids_pool;
#ifndef FB_EMU
  struct ProfEvent { int kind; cudaEvent_t a, b; };
  std::vector<ProfEvent> prof_events;
  cudaStream_t stream; cudaEvent_t ev0, ev1;
  struct StepGraph { cudaGraphExec_t exec; bool seen, failed; int n_sub; long long launches; DevData d; DevModel m; };
  StepGraph graph[2];          // [hold pending?]
  bool graphs_on;
#endif
};

// -------------------------------------------------------------------------------------------
// host / device seam: the one place that knows whether there is a device.  Under FB_EMU "device" memory is host memory, a copy
// is a memcpy that is done when it returns, and a launch runs its envs one after the other (emu_launch).
#ifndef FB_EMU
#define FB_CUDA_OK(call) do { cudaError_t err_ = (call); if (err_ != cudaSuccess) { s->err = std::string(#call) + ": " + cudaGetErrorString(err_); return -2; } } while (0)
static const char* const kVersion = "flybody_b200 0.2 (sm_90a)";
static void* dev_alloc(size_t bytes) {   // rare (create / first use): zero-fill and make it visible to every stream
  void* p = nullptr; if (cudaMalloc(&p, bytes ? bytes : 4) != cudaSuccess) return nullptr; cudaMemset(p, 0, bytes ? bytes : 4); cudaDeviceSynchronize(); return p; }
static void dev_free(void* p) { cudaFree(p); }
static int dev_open(FbSim* s, int n_envs) {
  if (cudaSetDevice(s->device) != cudaSuccess) return -2;
  cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking);
  cudaEventCreate(&s->ev0); cudaEventCreate(&s->ev1);
  s->graphs_on = getenv("FB_NO_GRAPH") == nullptr;
  // small batches are latency-bound (a per-CTA copy of the sweep program in shared memory halves the sweeps' latency);
  // at full occupancy the copy costs more than it saves and the compact program is read in place.  FB_BLOB=0/1 overrides.
  s->blob_in_smem = getenv("FB_BLOB") ? atoi(getenv("FB_BLOB")) : (n_envs <= 1024);
  return 0;
}
static void dev_close(FbSim* s) {
  cudaSetDevice(s->device); cudaStreamSynchronize(s->stream);
  for (auto& g : s->graph) if (g.exec) cudaGraphExecDestroy(g.exec);
  cudaEventDestroy(s->ev0); cudaEventDestroy(s->ev1); cudaStreamDestroy(s->stream);
}
static void dev_select(FbSim* s) { cudaSetDevice(s->device); }
// stream-ordered copies in any direction (the handle's stream is non-blocking: legacy default-stream copies would not order with
// its kernels); copy_rows_async moves `rows` rows of `width` bytes, `spitch` bytes apart in the source and `dpitch` in the destination
static int copy_async(FbSim* s, void* dst, const void* src, size_t bytes) {
  FB_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, s->stream));
  return 0;
}
static int copy_rows_async(FbSim* s, void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t rows) {
  FB_CUDA_OK(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, rows, cudaMemcpyDefault, s->stream));
  return 0;
}
static int sync_stream(FbSim* s) {
  FB_CUDA_OK(cudaStreamSynchronize(s->stream));
  FB_CUDA_OK(cudaGetLastError());
  return 0;
}
static int launch_check(FbSim* s, const char* who) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { s->err = std::string(who) + ": kernel launch failed (" + cudaGetErrorString(e) + ")"; return -2; }
  return 0;
}
static size_t dev_free_bytes() {      // (no answer: no limit)
  size_t free_b = 0, total_b = 0;
  return cudaMemGetInfo(&free_b, &total_b) == cudaSuccess ? free_b : std::numeric_limits<size_t>::max();
}
#else
static const char* const kVersion = "flybody_b200 0.2 (host emulation build: tests only)";
static void* dev_alloc(size_t bytes) { return calloc(bytes ? bytes : 4, 1); }
static void dev_free(void* p) { free(p); }
static int dev_open(FbSim*, int) { return 0; }
static void dev_close(FbSim*) {}
static void dev_select(FbSim*) {}
static int copy_async(FbSim*, void* dst, const void* src, size_t bytes) { memcpy(dst, src, bytes); return 0; }
static int copy_rows_async(FbSim*, void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t rows) {
  for (size_t r = 0; r < rows; r++) memcpy((char*)dst + r * dpitch, (const char*)src + r * spitch, width);
  return 0;
}
static int sync_stream(FbSim*) { return 0; }
static int launch_check(FbSim*, const char*) { return 0; }
static size_t dev_free_bytes() { return std::numeric_limits<size_t>::max(); }
// One emulated launch: the envs of [0, n), or of the list `ids`, one after the other, each through a zeroed slice exactly as large
// as the GPU launch makes a warp's shared memory, followed by a canary: a kernel that writes past its slice (on the GPU: into the
// next warp's slice or out of the block's allocation) aborts the CPU tests instead of passing.
template <typename Body> static void emu_launch(FbSim* s, const char* kernel, size_t slice, int n, const int* ids, Body body) {
  std::vector<unsigned char> buf(slice + 256, 0);
  memset(buf.data() + slice, 0xAB, 256);
  for (int k = 0; k < n; k++) body(buf.data(), ids ? ids[k] : k);
  for (size_t i = 0; i < 256; i++)
    if (buf[slice + i] != 0xAB) { fprintf(stderr, "fb_emu: shared-memory slice overrun in the %s kernel (slice %zu bytes)\n", kernel, slice); abort(); }
  s->launches++;
}
#endif
// a copy whose source the caller may reuse (or whose destination it reads) once the call returns
static int copy_sync(FbSim* s, void* dst, const void* src, size_t bytes) {
  const int rc = copy_async(s, dst, src, bytes);
  return rc != 0 ? rc : sync_stream(s);
}
// the outputs of a read, host or device: `rows` rows of `width` bytes, `spitch` bytes apart in the source and packed in the destination
// (spitch 0: a contiguous array, one row); a NULL destination is skipped.  The stream is idle when it returns.
struct ReadOut { void* dst; const void* src; size_t spitch, width, rows; };
static int read_out(FbSim* s, const std::vector<ReadOut>& outs) {
  for (const ReadOut& o : outs)
    if (o.dst && o.width && copy_rows_async(s, o.dst, o.width, o.src, o.spitch ? o.spitch : o.width, o.width, o.rows) != 0) return -2;
  return sync_stream(s);
}

static size_t slice_bytes(size_t fixed, size_t dyn_floats) { return ((((fixed + 15) & ~(size_t)15) + dyn_floats * sizeof(float)) + 15) & ~(size_t)15; }
// kernel = sequence of stages for one env.  Ph<f>: per-lane phase f(m, d, sh, e, y), a warp barrier follows;
// Wf<f>: warp function f(m, d, sh, e) written with WPAR sections (its own barriers inside).
template <auto F> struct Ph {
#ifdef __CUDACC__
  template <typename Sh> static __device__ __forceinline__ void run(const DevModel& m, const DevData& d, Sh& sh, int e, int y) { F(m, d, sh, e, y); }
#endif
  template <typename Sh> static void emu(const DevModel& m, const DevData& d, Sh& sh, int e) { for (int y = 0; y < FB_NY; y++) F(m, d, sh, e, y); }
};
template <auto F> struct Wf {
#ifdef __CUDACC__
  template <typename Sh> static __device__ __forceinline__ void run(const DevModel& m, const DevData& d, Sh& sh, int e, int) { F(m, d, sh, e); }
#endif
  template <typename Sh> static void emu(const DevModel& m, const DevData& d, Sh& sh, int e) { F(m, d, sh, e); }
};
#ifndef FB_EMU
// one warp per env: threadIdx.x = lane ("y" of the phase functions), threadIdx.y = env within the block
template <typename Sh> __device__ __forceinline__ void set_prog(Sh&, const unsigned*) {}
__device__ __forceinline__ void set_prog(ShTree& sh, const unsigned* p) { sh.prog = p; }
template <typename Sh> __device__ __forceinline__ void set_slice(Sh&, int) {}
__device__ __forceinline__ void set_slice(ShCol& sh, int slice) { sh.slice = slice; }
// e0 (the first env of the launch) is always 0.  It stays a run-time kernel parameter because ptxas (CUDA 12.9) schedules
// the step kernels differently without it: the velocity kernel grew by 104 SASS instructions and ran 3 % slower on an
// H100 SXM at 700 W.
template <typename Sh, typename... St>
__global__ void __launch_bounds__(32 * FB_WPB, FB_MINB) fb_run(DevModel m, DevData d, int slice, int e0, int nwarps, int blob_words) {
  extern __shared__ __align__(16) unsigned char fb_smem[];
  // optional CTA-wide copy of the sweep program in front of the warps' slices (the only block-level barrier of the step)
  unsigned* blob = reinterpret_cast<unsigned*>(fb_smem);
  if (blob_words) {
    for (int i = threadIdx.y * 32 + threadIdx.x; i < blob_words; i += 32 * FB_WPB) blob[i] = m.tsolve_blob[i];
    __syncthreads();
  }
  int e = e0 + blockIdx.x * FB_WPB + threadIdx.y;
  if (e >= e0 + nwarps) return;
  Sh& sh = *reinterpret_cast<Sh*>(fb_smem + (size_t)blob_words * 4 + (size_t)threadIdx.y * slice);
  int y = threadIdx.x;
  set_slice(sh, slice);
  if (blob_words) { set_prog(sh, blob); __syncwarp(); } else { set_prog(sh, m.tsolve_blob); __syncwarp(); }   // no CTA copy: read the program in place
#ifdef FB_CLK
  // latency profile: stage boundaries of env 0's warp, 32 slots per launch (slot 0 = kernel entry)
  int ci = 0; long long* ck = d.clk + 32 * d.clk_launch;
  if (e == 0 && y == 0) ck[ci] = clock64();
  ((St::run(m, d, sh, e, y), __syncwarp(), (e == 0 && y == 0 ? (void)(ck[++ci] = clock64()) : (void)0)), ...);
#else
  ((St::run(m, d, sh, e, y), __syncwarp()), ...);
#endif
}
// a step-stage launch on the handle's stream, between a pair of events while fb_profile is on
template <typename L> static void dev_launch(FbSim* s, int kind, L launch) {
#ifdef FB_CLK
  s->d.clk_launch = (int)(s->launches % 4096);
#endif
  if (s->prof_on) {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    cudaEventRecord(a, s->stream);
    launch();
    cudaEventRecord(b, s->stream);
    s->prof_events.push_back({kind, a, b});
  } else {
    launch();
  }
  s->launches++;
}
static void prof_collect(FbSim* s) {      // the recorded launches into prof_ms / prof_n (the stream is idle)
  for (auto& ev : s->prof_events) { float t = 0; cudaEventElapsedTime(&t, ev.a, ev.b); s->prof_ms[ev.kind] += t; s->prof_n[ev.kind]++; cudaEventDestroy(ev.a); cudaEventDestroy(ev.b); }
  s->prof_events.clear();
}
template <typename Sh, typename... St>
static void fb_launch(FbSim* s, int kind, size_t dyn_floats = 0, int nwarps = -1, int blob_words = 0) {
  if (nwarps < 0) nwarps = s->d.Np;          // step kernels cover the padded batch
  dim3 block(32, FB_WPB), grid((nwarps + FB_WPB - 1) / FB_WPB);
  size_t slice = slice_bytes(sizeof(Sh), dyn_floats), bytes = slice * FB_WPB + (size_t)blob_words * 4;
  static size_t configured = 0;
  if (bytes > configured) { cudaFuncSetAttribute(fb_run<Sh, St...>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes); configured = bytes; }
  dev_launch(s, kind, [&] { fb_run<Sh, St...><<<grid, block, bytes, s->stream>>>(s->m, s->d, (int)slice, 0, nwarps, blob_words); });
}
__global__ void __launch_bounds__(32 * FB_SOLVE_WPB, FB_MINB) fb_run_solve(DevModel m, DevData d, int nwarps) {
  extern __shared__ __align__(16) float fb_smem_w[];
  int e = blockIdx.x * FB_SOLVE_WPB + threadIdx.y;
  if (e >= nwarps) return;
#ifdef FB_CLK
  if (e == 0 && threadIdx.x == 0) d.clk[32 * d.clk_launch] = clock64();
#endif
  ksolve_warp(m, d, fb_smem_w + (size_t)threadIdx.y * FB_SOLVE_WARP_FLOATS, e);
#ifdef FB_CLK
  if (e == 0 && threadIdx.x == 0) d.clk[32 * d.clk_launch + 1] = clock64();
#endif
}
static void fb_launch_warp(FbSim* s, int kind) {
  dim3 block(32, FB_SOLVE_WPB), grid((s->d.Np + FB_SOLVE_WPB - 1) / FB_SOLVE_WPB);
  size_t bytes = sizeof(float) * FB_SOLVE_WARP_FLOATS * FB_SOLVE_WPB;
  static bool configured = false;
  if (!configured) { cudaFuncSetAttribute(fb_run_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes); configured = true; }
  dev_launch(s, kind, [&] { fb_run_solve<<<grid, block, bytes, s->stream>>>(s->m, s->d, s->d.Np); });
}
// one warp per problem w of [0, n), with `slice` bytes of shared memory each: k(slice, w).  K carries the kernel's parameters.  Slices
// are whole 16-byte units; saying so keeps the IK kernel's shared-memory addressing (and its registers) as it was without the launcher.
template <typename K> __global__ void __launch_bounds__(32 * FB_WPB) fb_run_warps(K k, int n, unsigned slice) {
  extern __shared__ __align__(16) unsigned char fb_smem_q[];
  const int w = blockIdx.x * FB_WPB + threadIdx.y;
  if (w < n) k(static_cast<unsigned char*>(__builtin_assume_aligned(fb_smem_q + (size_t)threadIdx.y * slice, 16)), w);
}
template <typename K> static void warp_launch(FbSim* s, const char*, int n, size_t slice, const K& k) {
  dev_launch(s, K_MISC, [&] { fb_run_warps<<<(n + FB_WPB - 1) / FB_WPB, dim3(32, FB_WPB), slice * FB_WPB, s->stream>>>(k, n, (unsigned)slice); });
}
#else
template <typename Sh> static void set_prog(Sh&, const unsigned*) {}
static void set_prog(ShTree& sh, const unsigned* p) { sh.prog = p; }
static void prof_collect(FbSim*) {}
// the stage list St over the envs of [0, n) or of the list `ids`
template <typename Sh, typename... St> static void emu_stages(FbSim* s, int kind, size_t dyn_floats, int n, const int* ids) {
  emu_launch(s, kKindNames[kind], slice_bytes(sizeof(Sh), dyn_floats), n, ids, [&](unsigned char* buf, int e) {
    Sh& sh = *reinterpret_cast<Sh*>(buf);
    set_prog(sh, s->m.tsolve_blob);        // host emulation: the program is read in place
    (St::emu(s->m, s->d, sh, e), ...);
  });
}
template <typename Sh, typename... St>
static void fb_launch(FbSim* s, int kind, size_t dyn_floats = 0, int nwarps = -1, int = 0) {
  emu_stages<Sh, St...>(s, kind, dyn_floats, nwarps < 0 ? s->d.Np : nwarps, nullptr);
}
static void fb_launch_warp(FbSim* s, int kind) {
  emu_launch(s, kKindNames[kind], sizeof(float) * FB_SOLVE_WARP_FLOATS, s->d.Np, nullptr,
             [&](unsigned char* buf, int e) { ksolve_warp(s->m, s->d, reinterpret_cast<float*>(buf), e); });
}
template <typename K> static void warp_launch(FbSim* s, const char* kernel, int n, size_t slice, const K& k) { emu_launch(s, kernel, slice, n, nullptr, k); }
#endif

// per-env kernels wrapped as single-phase functions
FB_DEV void ph_reset_scatter(const DevModel& m, const DevData& d, ShNone&, int e, int y) { kreset_scatter(m, d, e, y); }
FB_DEV void ph_reset_draw(const DevModel& m, const DevData& d, ShNone&, int w, int y) { if (w < d.rst_n) kprm_draw(m, d, d.rst_ids[w], y); }
FB_DEV void ph_reset_count(const DevModel&, const DevData& d, ShNone&, int w, int y) { if (w < d.rst_n) kprm_count(d, d.rst_ids[w], y); }
FB_DEV void ph_scatter(const DevModel& m, const DevData& d, ShNone&, int e, int y) { kscatter(m, d, e, y); }
FB_DEV void ph_clear_hold(const DevModel& m, const DevData& d, ShNone&, int e, int y) { kclear_hold(m, d, e, y); }
FB_DEV void ph_task_reset(const DevModel& m, const DevData& d, ShNone&, int e, int y) { ktask_reset(m, d, e, y); }
FB_DEV void ph_task_reset2(const DevModel& m, const DevData& d, ShNone&, int e, int y) { ktask_reset2(m, d, e, y); }
FB_DEV void ph_task_reset3(const DevModel& m, const DevData& d, ShNone&, int e, int y) { ktask_reset3(m, d, e, y); }
FB_DEV void ph_task_reset4(const DevModel& m, const DevData& d, ShNone&, int e, int y) { ktask_reset4(m, d, e, y); }
FB_DEV void ph_task_reset5(const DevModel& m, const DevData& d, ShNone&, int e, int y) { ktask_reset5(m, d, e, y); }
FB_DEV void ph_task_reward(const DevModel& m, const DevData& d, ShNone&, int e, int y) { ktask_reward(m, d, e, y); }
FB_DEV void ph_task_before(const DevModel& m, const DevData& d, ShNone&, int e, int y) { ktask_before(m, d, e, y); }
FB_DEV void ph_task_commit(const DevModel& m, const DevData& d, ShNone&, int e, int y) { ktask_commit(m, d, e, y); }
FB_DEV void ph_task_after(const DevModel& m, const DevData& d, ShNone&, int e, int y) { ktask_after(m, d, e, y); }
FB_DEV void ph_pack(const DevModel& m, const DevData& d, ShNone&, int e, int y) { kpack(m, d, e, y, d.nsub_done > 0 ? 1.0f / d.nsub_done : 1.0f); ktaskobs(m, d, e, y); }
// Smooth dynamics in half-solve form: with M = L^T D L and u = L^-T qfrc_smooth,
//   J qacc_smooth = Z (D^-1/2 u)          (Z = D^-1/2 L^-T J^T, rows written by the projection kernel)
//   qacc          = L^-1 (D^-1 u + D^-1/2 Z^T f)
// so the step needs L^-T once (here) and L^-1 once (finish kernel) instead of two full solves.  qtmp <- D^-1 u,
// dof_isd <- D^-1/2, XS <- D^-1/2 u for kref.
FB_WARPFN void wf_smooth_solve(const DevModel& m, const DevData& d, ShTree& sh, int e) { tsolve_a(m, d, sh, e); }
FB_DEV void ph_smooth_out(FB_PHASE_ARGS) {
  float* xs = sh_dyn(sh); const float* lds = xs + FB_NXS(m);
  for (int i = y; i < m.nv; i += FB_NY) {
    float D = LDS(m.dof_Madr[i]), u = XS(i), isd = 1.0f / sqrtf(D);
    AT(d.qtmp, i) = u / D; AT(d.dof_isd, i) = isd; XS(i) = u * isd;
  }
}

// the stage lists of the seven step kernels (also named by step_kernel_fn for the occupancy query)
#define FB_ST_POS Ph<kpos_p0>, Ph<kpos_p1>, Ph<kpos_p1b>, Ph<kpos_p2>, Ph<kpos_p3>, Ph<kpos_p3b>, Ph<kpos_p4>, Wf<kpos_factor>, Ph<kpos_p6w>, Ph<kpos_p6d>, Wf<kpos_factor>, Ph<kpos_p9>
#define FB_ST_COL Ph<kcol_stage>, Wf<kcol_broad>, Ph<kcol_narrow>, Wf<kcol_mpr>, Ph<kcol_compact>
#define FB_ST_PROJ Ph<kcon_p0>, Ph<kcon_p1>, Ph<kcon_p2>, Ph<kcon_p3>, Ph<kproj_p0>, Ph<kproj_p1>
#define FB_ST_VEL Ph<kvel_p0>, Ph<kvel_p1>, Ph<kvel_p1b<false>>, Ph<kvel_p2>, Ph<kvel_p3>, Ph<kvel_p3b>, Ph<kvel_p4>
#define FB_ST_VEL_PRM Ph<kvel_p0>, Ph<kvel_p1>, Ph<kvel_p1b<true>>, Ph<kvel_p2>, Ph<kvel_p3>, Ph<kvel_p3b>, Ph<kvel_p4>    // with a parameter overlay
#define FB_ST_SMOOTH Ph<kact_p0>, Ph<kact_p1>, Ph<kact_p2>, Ph<kact_p2b>, Ph<kact_p3>, Wf<wf_smooth_solve>, Ph<ph_smooth_out>, Ph<kref>
#define FB_ST_FINISH Ph<kfin_f1>, Wf<kfin_solve>, Ph<kfin_f5>, Ph<kfin_f6>, Ph<kfin_f7>, Wf<kfin_solve_euler>, Ph<kfin_f8>, Ph<kfin_f9>, Ph<kfin_f10>
static size_t dyn_pos(const DevModel& m) { return (size_t)FB_PARTF + std::max((size_t)m.nM, (size_t)10 * m.nbody); }   // LS region: inertia matrix rows, before that the composite inertias (CRBS)
static size_t dyn_col(const DevModel& m) { return (size_t)FB_COL_DYN(m); }
static size_t dyn_proj(const DevModel&) { return (size_t)FB_NY * FB_ZCAP; }
static size_t dyn_vel(const DevModel&) { return (size_t)FB_PARTF; }
static size_t dyn_tsolve(const DevModel& m) { return (size_t)(FB_NXS(m) + ((m.nM + 3) & ~3)); }

// Heightfield contacts: DevHf travels in its own kernel (not in DevModel / DevData: the step kernels of models without a
// heightfield keep their parameter layout).  launch_hfield covers the envs of [0, n) or of a device list, as fb_launch_ids does
// for the position / velocity stage (fb_state_load recomputes what a state row does not carry), through the stage functions of
// the step kernels.  One env per block: the collision stage pools the jobs of a block's envs on warp 0 and takes them to be
// consecutive envs, so a listed env runs as warp 0 of a block whose other slices report no jobs.
#ifndef FB_EMU
__global__ void __launch_bounds__(32 * FB_WPB, FB_MINB) fb_hf_kernel(DevModel m, DevData d, DevHf p, int nwarps) {
  const int e = blockIdx.x * FB_WPB + threadIdx.y;
  if (e >= nwarps) return;
  khf_narrow(m, d, p, e, threadIdx.x); __syncwarp();
  khf_append(m, d, p, e, threadIdx.x);
}
template <typename Sh, typename... St>
__global__ void __launch_bounds__(32 * FB_WPB, FB_MINB) fb_run_ids(DevModel m, DevData d, int slice, const int* ids) {
  extern __shared__ __align__(16) unsigned char fb_smem[];
  for (int i = threadIdx.x; i < (FB_WPB - 1) * slice / 4; i += 32) reinterpret_cast<unsigned*>(fb_smem + slice)[i] = 0u;
  const int e = ids[blockIdx.x], y = threadIdx.x;
  Sh& sh = *reinterpret_cast<Sh*>(fb_smem);
  set_slice(sh, slice); set_prog(sh, m.tsolve_blob); __syncwarp();
  ((St::run(m, d, sh, e, y), __syncwarp()), ...);
}
__global__ void __launch_bounds__(32 * FB_WPB, FB_MINB) fb_hf_kernel_ids(      // (the bounds of fb_hf_kernel: the same code)
DevModel m, DevData d, DevHf p, const int* ids) {
  const int e = ids[blockIdx.x];
  khf_narrow(m, d, p, e, threadIdx.x); __syncwarp();
  khf_append(m, d, p, e, threadIdx.x);
}
static void launch_hfield(FbSim* s, const int* ids, int n) {
  if (ids) fb_hf_kernel_ids<<<n, 32, 0, s->stream>>>(s->m, s->d, s->hf, ids);
  else fb_hf_kernel<<<(n + FB_WPB - 1) / FB_WPB, dim3(32, FB_WPB), 0, s->stream>>>(s->m, s->d, s->hf, n);
  s->launches++;
}
template <typename Sh, typename... St>
static void fb_launch_ids(FbSim* s, int, size_t dyn_floats, const int* ids, int n) {
  const size_t slice = slice_bytes(sizeof(Sh), dyn_floats), bytes = slice * FB_WPB;
  static size_t configured = 0;
  if (bytes > configured) { cudaFuncSetAttribute(fb_run_ids<Sh, St...>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes); configured = bytes; }
  fb_run_ids<Sh, St...><<<n, dim3(32, 1), bytes, s->stream>>>(s->m, s->d, (int)slice, ids);
  s->launches++;
}
static const void* step_kernel_fn(int kind, bool prm) {
  switch (kind) {
    case K_SMOOTH: return (const void*)fb_run<ShTree, FB_ST_SMOOTH>;
    case K_SOLVE: return (const void*)fb_run_solve;
    case K_FINISH: return (const void*)fb_run<ShTree, FB_ST_FINISH>;
    case K_POS: return (const void*)fb_run<ShTree, FB_ST_POS>;
    case K_COL: return (const void*)fb_run<ShCol, FB_ST_COL>;
    case K_PROJ: return (const void*)fb_run<ShCon, FB_ST_PROJ>;
    case K_VEL: return prm ? (const void*)fb_run<ShTree, FB_ST_VEL_PRM> : (const void*)fb_run<ShTree, FB_ST_VEL>;
    default: return nullptr;
  }
}
// the occupancy query of fb_step_kernel_smem (0 under emulation)
static int step_kernel_blocks_per_sm(FbSim* s, int kind, size_t bytes, int* blocks) {
  FB_CUDA_OK(cudaSetDevice(s->device));
  FB_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks, step_kernel_fn(kind, s->d.prm != nullptr), 32 * FB_WPB, bytes));
  return 0;
}
#else
static void launch_hfield(FbSim* s, const int* ids, int n) {
  emu_launch(s, "hfield", 0, n, ids, [&](unsigned char*, int e) {
    for (int y = 0; y < FB_NY; y++) khf_narrow(s->m, s->d, s->hf, e, y);
    for (int y = 0; y < FB_NY; y++) khf_append(s->m, s->d, s->hf, e, y);
  });
}
template <typename Sh, typename... St>
static void fb_launch_ids(FbSim* s, int kind, size_t dyn_floats, const int* ids, int n) { emu_stages<Sh, St...>(s, kind, dyn_floats, n, ids); }
static int step_kernel_blocks_per_sm(FbSim*, int, size_t, int* blocks) { *blocks = 0; return 0; }
#endif

static void launch_step1(FbSim* s) {
  fb_launch<ShTree, FB_ST_POS>(s, K_POS, dyn_pos(s->m));
  fb_launch<ShCol, FB_ST_COL>(s, K_COL, dyn_col(s->m));
  if (s->hf_on) launch_hfield(s, nullptr, s->d.N);     // heightfield contacts join the contact list before the constraint rows are built
  fb_launch<ShCon, FB_ST_PROJ>(s, K_PROJ, dyn_proj(s->m));
  if (s->d.prm) fb_launch<ShTree, FB_ST_VEL_PRM>(s, K_VEL, dyn_vel(s->m));
  else fb_launch<ShTree, FB_ST_VEL>(s, K_VEL, dyn_vel(s->m));
}
static void launch_step1_ids(FbSim* s, const int* ids, int n) {      // ids: a device list
  fb_launch_ids<ShTree, FB_ST_POS>(s, K_POS, dyn_pos(s->m), ids, n);
  fb_launch_ids<ShCol, FB_ST_COL>(s, K_COL, dyn_col(s->m), ids, n);
  if (s->hf_on) launch_hfield(s, ids, n);
  fb_launch_ids<ShCon, FB_ST_PROJ>(s, K_PROJ, dyn_proj(s->m), ids, n);
  if (s->d.prm) fb_launch_ids<ShTree, FB_ST_VEL_PRM>(s, K_VEL, dyn_vel(s->m), ids, n);
  else fb_launch_ids<ShTree, FB_ST_VEL>(s, K_VEL, dyn_vel(s->m), ids, n);
}
static void launch_step2(FbSim* s, bool integrate) {
  s->d.do_integrate = integrate ? 1 : 0;     // read by the solve (warm-start bookkeeping) and the finish kernel
  fb_launch<ShTree, FB_ST_SMOOTH>(s, K_SMOOTH, dyn_tsolve(s->m), -1, s->blob_in_smem ? s->m.ts_blob_words : 0);
  fb_launch_warp(s, K_SOLVE);
  fb_launch<ShTree, FB_ST_FINISH>(s, K_FINISH, dyn_tsolve(s->m), -1, s->blob_in_smem ? s->m.ts_blob_words : 0);
}

// -------------------------------------------------------------------------------------------
// model upload
template <typename T> static const T* up(FbSim* s, const std::vector<T>& v) {
  void* p = dev_alloc(sizeof(T) * std::max<size_t>(v.size(), 1));
  if (p && v.size() && copy_sync(s, p, v.data(), sizeof(T) * v.size()) != 0) { dev_free(p); p = nullptr; }   // a failed upload is a missing buffer
  s->allocs.push_back(p);
  return (const T*)p;
}
static const float* upf(FbSim* s, const double* src, size_t n) { std::vector<float> v(n); for (size_t i = 0; i < n; i++) v[i] = (float)src[i]; return up(s, v); }
static const float* upf3(FbSim* s, const double* src, size_t n) {      // n 3-vectors, padded to four floats each (fb_math.h: mld3)
  std::vector<float> v(4 * std::max<size_t>(n, 1), 0.0f);
  for (size_t i = 0; i < n; i++) for (int k = 0; k < 3; k++) v[4 * i + k] = (float)src[3 * i + k];
  return up(s, v);
}
static const int* upi(FbSim* s, const int32_t* src, size_t n) { std::vector<int> v(src, src + n); return up(s, v); }
template <typename T> static T* dalloc(FbSim* s, size_t n) { void* p = dev_alloc(sizeof(T) * n); s->allocs.push_back(p); return (T*)p; }
// free the buffers a replaced program owned (the stream is idle: the callers synchronise first)
static void scope_free(FbSim* s, std::vector<void*>& scope) {
  for (void* p : scope) { s->allocs.erase(std::find(s->allocs.begin(), s->allocs.end(), p)); dev_free(p); }
  scope.clear();
}
// the buffers `alloc` allocates (dalloc / up) become `scope`; if one of them is missing the whole group is freed again and the
// call fails with `oom` as its message
template <typename F> static int scope_alloc(FbSim* s, std::vector<void*>& scope, const char* oom, F alloc) {
  const size_t mark = s->allocs.size();
  alloc();
  scope.assign(s->allocs.begin() + mark, s->allocs.end());
  for (void* p : scope) if (!p) { scope_free(s, scope); s->err = oom; return -4; }
  return 0;
}
// one pool for `rows` rows (`unit` says what a row is) of `row_bytes` bytes, made by alloc(rows) unless `cap` rows fit already
template <typename F> static int grow(FbSim* s, const char* who, Pool& pool, size_t rows, size_t row_bytes, const char* what, const char* unit, F alloc) {
  if (rows <= pool.cap) return 0;
  if (sync_stream(s) != 0) return -2;
  scope_free(s, pool.bufs); pool.cap = 0;
  if (rows * row_bytes > dev_free_bytes()) {
    s->err = std::string(who) + ": the " + what + " of " + std::to_string(rows) + " rows (" + unit + ") do not fit the device's free memory"; return -4; }
  const std::string oom = std::string(who) + ": out of device memory (" + what + ")";
  if (int rc = scope_alloc(s, pool.bufs, oom.c_str(), [&] { alloc(rows); })) return rc;
  pool.cap = rows;
  return 0;
}

static int build_model(FbSim* s, const FbModel* h) {
  DevModel& m = s->m;
  memset(&m, 0, sizeof(m));
  m.nq = h->nq; m.nv = h->nv; m.nu = h->nu; m.na = h->na; m.nbody = h->nbody; m.njnt = h->njnt; m.ngeom = h->ngeom;
  m.npair = h->npair; m.nsite = h->nsite; m.ntendon = h->ntendon; m.nwrap = h->nwrap; m.nsensor = h->nsensor;
  m.nsensordata = h->nsensordata; m.nM = h->nM; m.nfluid = h->nfluid;
  m.noslip_iterations = h->opt_noslip_iterations; m.cone_elliptic = h->opt_cone_elliptic; m.ls_tolerance = 1e-3f;
  // solver limits = the model's own (mjOption iterations / ls_iterations: 100 / 50 for the fly, fruitfly.xml:4 leaves the defaults);
  // the loops leave on convergence long before (1-4 Newton iterations, 2-4 line-search evaluations per substep in the walking workload)
  m.max_iter = h->opt_iterations > 0 ? h->opt_iterations : 100; m.ls_iter = h->opt_ls_iterations > 0 ? h->opt_ls_iterations : 50;
  if (h->nv > 4 * FB_SOLVE_NCAP) { s->err = "nv exceeds the solver's per-dof accumulator window (4 * FB_SOLVE_NCAP)"; return -3; }
  // actuation (kact_p1) implements a fixed gain, bias none (0) or affine (1), and dynamics none (0) or filter (2: act += h * act_dot,
  // Euler); any other type, e.g. filterexact (3), would be stepped as a plain filter, so such a model is refused here
  for (int i = 0; i < h->nu; i++) {
    int dt = h->actuator_dyntype[i], bt = h->actuator_biastype[i], aa = h->actuator_actadr[i];
    std::string who = "actuator " + std::to_string(i) + ": ";
    if (dt != 0 && dt != 2) { s->err = who + "dyntype " + std::to_string(dt) + " is not implemented (none = 0, filter = 2 are)"; return -3; }
    if (bt != 0 && bt != 1) { s->err = who + "biastype " + std::to_string(bt) + " is not implemented (none = 0, affine = 1 are)"; return -3; }
    if ((dt == 2) != (aa >= 0) || aa >= h->na) { s->err = who + "activation address " + std::to_string(aa) + " does not match dyntype " + std::to_string(dt); return -3; }
  }
  // the touch ray test (kfin_f9, kinv_sensors) knows capsule sites and treats every other site as a sphere of radius size[0]: a touch
  // sensor on an ellipsoid, box or cylinder site would be tested against the wrong shape, so such a model is refused
  for (int i = 0; i < h->nsensor; i++) {
    if (h->sensor_type[i] != FB_SENS_TOUCH) continue;
    int t = h->site_type[h->sensor_objid[i]];
    if (t != FB_GEOM_SPHERE && t != FB_GEOM_CAPSULE) { s->err = "sensor " + std::to_string(i) + ": touch site of type " + std::to_string(t) + " is not implemented (sphere = 2, capsule = 3 are)"; return -3; }
  }
  { const char* rt = getenv("FB_SOLVE_RTOL"); m.solve_rtol = rt ? (float)atof(rt) : 1e-6f; }     // relative improvement that ends the Newton iteration (test hook)
  { const char* nc = getenv("FB_SOLVE_NCAP"); m.solve_ncap = nc ? atoi(nc) : FB_SOLVE_NCAP; if (m.solve_ncap > FB_SOLVE_NCAP) m.solve_ncap = FB_SOLVE_NCAP; }   // test hook: smaller cap -> global-memory path
  m.timestep = (float)h->opt_timestep; m.density = (float)h->opt_density; m.viscosity = (float)h->opt_viscosity;
  for (int i = 0; i < 3; i++) { m.gravity[i] = (float)h->opt_gravity[i]; m.wind[i] = (float)h->opt_wind[i]; }
  m.impratio = (float)h->opt_impratio; m.tolerance = (float)h->opt_tolerance; m.noslip_tolerance = (float)h->opt_noslip_tolerance;
  m.meaninertia = (float)h->stat_meaninertia;
  int nb = m.nbody, nv = m.nv;
  // ---- tree partition: roots = children of world; each root's child sub-trees are packed into lists
  std::vector<int> roots, isroot(nb, 0);
  for (int b = 1; b < nb; b++) if (h->body_parentid[b] == 0) { roots.push_back(b); isroot[b] = 1; }
  isroot[0] = 1;   // the world behaves like a root for "parent is root" tests (never accumulated into)
  for (int r : roots) {
    const int jt = h->body_jntnum[r] == 1 ? h->jnt_type[h->body_jntadr[r]] : -1;
    if (!(h->body_jntnum[r] == 0 || jt == FB_JNT_FREE || jt == FB_JNT_BALL)) { s->err = "root bodies must carry a single free or ball joint or none"; return -3; }
  }
  for (int j = 0; j < h->njnt; j++) {
    if (h->jnt_type[j] != FB_JNT_BALL) continue;
    // ball joints are stepped as the rotational half of a free joint: no quaternion spring, no cone limit (neither is implemented)
    if (h->body_parentid[h->jnt_bodyid[j]] != 0) { s->err = "ball joints are implemented on root bodies only"; return -3; }
    if (h->jnt_stiffness[j] != 0 || h->jnt_limited[j]) { s->err = "ball joints with stiffness or limits are not implemented"; return -3; }
  }
  for (int j = 0; j < h->njnt; j++)
    if (h->jnt_type[j] != FB_JNT_FREE && h->jnt_type[j] != FB_JNT_BALL && h->jnt_type[j] != FB_JNT_HINGE) { s->err = "joint type not implemented (free, ball and hinge are)"; return -3; }
  std::vector<std::vector<int>> subtrees; std::vector<int> sub_root;
  for (size_t ri = 0; ri < roots.size(); ri++) {
    for (int b = 1; b < nb; b++) if (h->body_parentid[b] == roots[ri]) {
      std::vector<int> st; std::vector<char> in(nb, 0); in[b] = 1; st.push_back(b);
      for (int c = b + 1; c < nb; c++) if (in[h->body_parentid[c]]) { in[c] = 1; st.push_back(c); }
      subtrees.push_back(st); sub_root.push_back((int)ri);
    }
  }
  size_t maxsz = 1, total = 0; for (auto& st : subtrees) { maxsz = std::max(maxsz, st.size()); total += st.size(); }
  int nlist = (int)std::min<size_t>(FB_NLMAX, std::max<size_t>(1, (total + maxsz - 1) / maxsz + 1));
  std::vector<std::vector<int>> lists(nlist); std::vector<int> lroot(nlist, -1);
  std::vector<size_t> order(subtrees.size()); for (size_t i = 0; i < order.size(); i++) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return subtrees[a].size() > subtrees[b].size(); });
  for (size_t oi : order) {
    int best = -1;
    for (int l = 0; l < nlist; l++) { if (lroot[l] != -1 && lroot[l] != sub_root[oi]) continue; if (best < 0 || lists[l].size() < lists[best].size()) best = l; }
    if (best < 0) { s->err = "tree partition: more roots with children than lists"; return -3; }
    lroot[best] = sub_root[oi];
    lists[best].insert(lists[best].end(), subtrees[oi].begin(), subtrees[oi].end());
  }
  std::vector<int> ladr, lnum, lbody, lr;
  for (int l = 0; l < nlist; l++) { ladr.push_back((int)lbody.size()); lnum.push_back((int)lists[l].size()); lbody.insert(lbody.end(), lists[l].begin(), lists[l].end()); lr.push_back(lroot[l] < 0 ? 0 : lroot[l]); }
  m.nroot = (int)roots.size(); m.nlist = nlist;
  // the dofs of each list in factorisation order (bodies in reverse, dofs in reverse): list l's are dl[dadr[l] .. dadr[l] + dnum[l]);
  // dof_list: the list a dof belongs to, -1 for root dofs
  std::vector<int> dadr, dnum, dl, dof_list(nv, -1);
  for (int l = 0; l < nlist; l++) { dadr.push_back((int)dl.size()); int c = 0;
    for (int bi = (int)lists[l].size() - 1; bi >= 0; bi--) { int bb = lists[l][bi]; for (int kk = h->body_dofnum[bb] - 1; kk >= 0; kk--) { dl.push_back(h->body_dofadr[bb] + kk); dof_list[h->body_dofadr[bb] + kk] = l; c++; } }
    dnum.push_back(c); m.max_list_ndof = std::max(m.max_list_ndof, c); }
  m.root_body = up(s, roots); m.list_adr = up(s, ladr); m.list_num = up(s, lnum); m.list_body = up(s, lbody); m.list_root = up(s, lr);
  m.body_isroot = up(s, isroot);
  { // bodies the acceleration-stage sensors need: force sensors read the subtree sum at the site's body;
    // accelerometers need the (delta) acceleration of the site's body; both need their ancestors' deltas
    std::vector<int> sfrc(nb, 0), sacc(nb, 0), frcroot(nb, 0);
    for (int t = 0; t < h->nsensor; t++) { int b = h->site_bodyid[h->sensor_objid[t]]; if (h->sensor_type[t] == FB_SENS_FORCE) frcroot[b] = 1; if (h->sensor_type[t] == FB_SENS_FORCE || h->sensor_type[t] == FB_SENS_ACCELEROMETER) sacc[b] = 1; }
    for (int b = 1; b < nb; b++) if (frcroot[b] || sfrc[h->body_parentid[b]]) sfrc[b] = 1;
    for (int b = 1; b < nb; b++) if (sfrc[b]) sacc[b] = 1;
    for (int b = nb - 1; b > 0; b--) if (sacc[b]) sacc[h->body_parentid[b]] = 1;
    sacc[0] = 0;
    m.body_sensacc = up(s, sacc); m.body_sensfrc = up(s, sfrc);
  }
  // geoms and sites come in body order (the compiler stores them so)
  for (int g = 1; g < m.ngeom; g++) if (h->geom_bodyid[g] < h->geom_bodyid[g - 1]) { s->err = "geoms not in body order"; return -3; }
  for (int t = 1; t < m.nsite; t++) if (h->site_bodyid[t] < h->site_bodyid[t - 1]) { s->err = "sites not in body order"; return -3; }
  // dof helpers
  std::vector<int> subend(nv), depth(nv), disroot(nv), chainlen(nv);
  for (int i = 0; i < nv; i++) subend[i] = i;
  for (int i = nv - 1; i >= 0; i--) { int p = h->dof_parentid[i]; if (p >= 0) subend[p] = std::max(subend[p], subend[i]); }
  for (int i = 0; i < nv; i++) {
    disroot[i] = isroot[h->dof_bodyid[i]] && h->dof_bodyid[i] != 0;
    int len = 0, nonroot = 0;
    for (int j = i; j >= 0; j = h->dof_parentid[j]) { len++; if (j != i && !(isroot[h->dof_bodyid[j]] && h->dof_bodyid[j] != 0)) nonroot++; }
    chainlen[i] = len;
    depth[i] = disroot[i] ? (i - h->body_dofadr[h->dof_bodyid[i]]) : nonroot;
  }
  { std::vector<int> anc(h->nM, -1); for (int i = 0; i < nv; i++) { int t = 0; for (int j = i; j >= 0; j = h->dof_parentid[j], t++) anc[h->dof_Madr[i] + t] = j; } m.dof_anc = up(s, anc); }
  { // the root a list dof hangs off, and which roots have lists
    std::vector<int> rootidx(nv, -1), haslists(roots.size(), 0);
    for (int i = 0; i < nv; i++) if (dof_list[i] >= 0) { rootidx[i] = lr[dof_list[i]]; haslists[lr[dof_list[i]]] = 1; }
    m.dof_rootidx = up(s, rootidx); m.root_haslists = up(s, haslists);
  }
  { // common-ancestor counts of every dof pair (kproj_p1: the dofs two constraint rows share are the common TAIL of their chains)
    if (nv > 255) { s->err = "too many dofs for the byte-sized common-ancestor table"; return -3; }
    if (nv > 128) { s->err = "too many dofs for the register-path force gather (4 dofs per lane, fb_solver_reg.h)"; return -3; }
    std::vector<unsigned char> lca((size_t)nv * nv, 0); std::vector<int> mark(nv, -1);
    for (int a = 0; a < nv; a++) {
      for (int j = a; j >= 0; j = h->dof_parentid[j]) mark[j] = a;
      for (int b = 0; b < nv; b++) { int j = b; while (j >= 0 && mark[j] != a) j = h->dof_parentid[j]; lca[(size_t)a * nv + b] = (unsigned char)(j >= 0 ? chainlen[j] : 0); }
    }
    m.dof_lca = up(s, lca);
  }
  { std::vector<int> adh(nb, -1); for (int i = 0; i < h->nu; i++) if (h->actuator_trntype[i] == FB_TRN_BODY) adh[h->actuator_trnid[i]] = i; m.body_adhesion = up(s, adh); }
  { // packed headers of the lock-step sweeps (see fb_tree.h), deepest-first (a) and shallowest-first (c)
    if (h->nM >= 4096 || nv >= 256) { s->err = "model too large for the packed sweep headers (nM < 4096, nv < 256)"; return -3; }
    std::vector<unsigned> ha((size_t)FB_NY * std::max(m.max_list_ndof, 1), 0xffffffffu), hc(ha);
    auto pack = [&](int k) -> unsigned {
      if (chainlen[k] >= 64 || depth[k] >= 64) return 0xfffffffeu;
      return (unsigned)h->dof_Madr[k] | ((unsigned)chainlen[k] << 12) | ((unsigned)depth[k] << 18) | ((unsigned)k << 24); };
    for (int l = 0; l < nlist && FB_FSUB * l + FB_FSUB <= FB_NY; l++) for (int st = 0; st < dnum[l]; st++) for (int u = 0; u < FB_FSUB; u++) {
      unsigned a = pack(dl[dadr[l] + st]), c = pack(dl[dadr[l] + dnum[l] - 1 - st]);
      if (a == 0xfffffffeu || c == 0xfffffffeu) { s->err = "chain too long for the packed sweep headers"; return -3; }
      ha[(size_t)st * FB_NY + FB_FSUB * l + u] = a; hc[(size_t)st * FB_NY + FB_FSUB * l + u] = c; }
    { // the headers + ancestor slots as bytes, in one blob that the smooth / finish kernels copy into shared memory
      if (nv + FB_ROOTD * nlist >= 256) { s->err = "too many dofs for byte-sized sweep slots"; return -3; }
      const int H = (int)ha.size(), nmp = (h->nM + 3) & ~3;
      std::vector<unsigned> blob((((size_t)2 * H + 2 * nmp / 4) + 3) & ~(size_t)3, 0u);       // whole 16-byte units: the warps' slices follow
      for (int i = 0; i < H; i++) { blob[i] = ha[i]; blob[H + i] = hc[i]; }
      unsigned char* b8 = reinterpret_cast<unsigned char*>(blob.data() + 2 * H);
      for (int i = 0; i < nv; i++) { int t = 0; for (int j = i; j >= 0; j = h->dof_parentid[j], t++) {
          // shared-memory slot of the t-th ancestor: root dofs map to the list's private accumulators
          int slot = (disroot[j] && dof_list[i] >= 0) ? nv + FB_ROOTD * dof_list[i] + depth[j] : j;
          b8[h->dof_Madr[i] + t] = (unsigned char)slot; b8[nmp + h->dof_Madr[i] + t] = (unsigned char)j; } }
      m.tsolve_blob = up(s, blob); m.ts_hdr_words = H; m.ts_nm_pad = nmp; m.ts_blob_words = (int)blob.size();
    }
    std::vector<int> ancadr(h->nM, 0);      // row address (dof_Madr) of the ancestor an entry of the packed factor belongs to
    for (int i = 0; i < nv; i++) { int t = 0; for (int j = i; j >= 0; j = h->dof_parentid[j], t++) ancadr[h->dof_Madr[i] + t] = h->dof_Madr[j]; }
    { // balanced schedule of the factorisation sweeps (fb_tree.h: factor_step_sched): the rank-1 update of one ancestor row by the
      // step's dof of one list is a work item (cost = its length + a constant); the items of a step touch different rows, so they
      // are dealt to the 32 lanes longest-first onto the least loaded lane instead of 3 fixed lanes per list
      const int nstep = std::max(m.max_list_ndof, 1);
      std::vector<unsigned> rng((size_t)FB_NY * nstep, 0u); std::vector<unsigned> items;
      for (int st = 0; st < nstep; st++) {
        struct It { unsigned x, y; int cost; };
        std::vector<It> its;
        for (int l = 0; l < nlist; l++) {
          if (st >= dnum[l]) continue;
          const int k = dl[dadr[l] + st], adrk = h->dof_Madr[k], len = chainlen[k];
          for (int t = 1; t < 1 + depth[k]; t++) its.push_back({(unsigned)adrk | ((unsigned)t << 12) | ((unsigned)(len - t) << 18), (unsigned)ancadr[adrk + t], len - t + 6});
        }
        std::stable_sort(its.begin(), its.end(), [](const It& a, const It& b) { return a.cost > b.cost; });
        std::vector<std::vector<It>> lane_items(FB_NY); std::vector<int> load(FB_NY, 0);
        for (const It& it : its) { int best = 0; for (int y = 1; y < FB_NY; y++) if (load[y] < load[best]) best = y; lane_items[best].push_back(it); load[best] += it.cost; }
        for (int y = 0; y < FB_NY; y++) {
          if (items.size() / 2 >= 65536 || lane_items[y].size() >= 65536) { s->err = "factorisation schedule too long"; return -3; }
          rng[(size_t)st * FB_NY + y] = (unsigned)(items.size() / 2) | ((unsigned)lane_items[y].size() << 16);
          for (const It& it : lane_items[y]) { items.push_back(it.x); items.push_back(it.y); }
        }
      }
      if (items.empty()) { items.push_back(0); items.push_back(0); }
      m.fs_rng = up(s, rng); m.fs_items = reinterpret_cast<const FsItem*>(up(s, items));
    }
  }
  { std::vector<float> mdamp(h->nM, 0.0f); for (int i = 0; i < nv; i++) mdamp[h->dof_Madr[i]] = (float)h->dof_damping[i]; m.M_damp = up(s, mdamp); }
  m.dof_subend = up(s, subend); m.dof_depth = up(s, depth); m.dof_chainlen = up(s, chainlen);
  // plain copies
  m.body_parentid = upi(s, h->body_parentid, nb);
  m.body_jntadr = upi(s, h->body_jntadr, nb); m.body_jntnum = upi(s, h->body_jntnum, nb);
  m.body_dofadr = upi(s, h->body_dofadr, nb); m.body_dofnum = upi(s, h->body_dofnum, nb);
  m.body_lastdof = upi(s, h->body_lastdof, nb); m.body_fluid_ellipsoid = upi(s, h->body_fluid_ellipsoid, nb);
  m.body_pos = upf3(s, h->body_pos, nb); m.body_quat = upf(s, h->body_quat, 4 * nb); m.body_ipos = upf3(s, h->body_ipos, nb);
  m.body_iquat = upf(s, h->body_iquat, 4 * nb); m.body_mass = upf(s, h->body_mass, nb); m.body_inertia = upf3(s, h->body_inertia, nb);
  m.body_invweight0 = upf(s, h->body_invweight0, 2 * nb);
  int nj = m.njnt;
  m.jnt_type = upi(s, h->jnt_type, nj); m.jnt_qposadr = upi(s, h->jnt_qposadr, nj); m.jnt_dofadr = upi(s, h->jnt_dofadr, nj);
  m.jnt_bodyid = upi(s, h->jnt_bodyid, nj); m.jnt_limited = upi(s, h->jnt_limited, nj);
  m.jnt_pos = upf3(s, h->jnt_pos, nj); m.jnt_axis = upf3(s, h->jnt_axis, nj); m.jnt_stiffness = upf(s, h->jnt_stiffness, nj);
  m.jnt_range = upf(s, h->jnt_range, 2 * nj); m.jnt_solref = upf(s, h->jnt_solref, 2 * nj); m.jnt_solimp = upf(s, h->jnt_solimp, 5 * nj);
  m.jnt_margin = upf(s, h->jnt_margin, nj); m.qpos0 = upf(s, h->qpos0, m.nq); m.qpos_spring = upf(s, h->qpos_spring, m.nq);
  m.dof_bodyid = upi(s, h->dof_bodyid, nv); m.dof_jntid = upi(s, h->dof_jntid, nv); m.dof_parentid = upi(s, h->dof_parentid, nv);
  m.dof_Madr = upi(s, h->dof_Madr, nv); m.dof_armature = upf(s, h->dof_armature, nv); m.dof_damping = upf(s, h->dof_damping, nv);
  m.dof_invweight0 = upf(s, h->dof_invweight0, nv);
  int ng = m.ngeom;
  m.geom_type = upi(s, h->geom_type, ng); m.geom_bodyid = upi(s, h->geom_bodyid, ng); m.geom_condim = upi(s, h->geom_condim, ng);
  m.geom_size = upf3(s, h->geom_size, ng); m.geom_pos = upf3(s, h->geom_pos, ng); m.geom_quat = upf(s, h->geom_quat, 4 * ng);
  m.geom_rbound = upf(s, h->geom_rbound, ng); m.geom_friction = upf(s, h->geom_friction, 3 * ng); m.geom_solmix = upf(s, h->geom_solmix, ng);
  m.geom_solref = upf(s, h->geom_solref, 2 * ng); m.geom_solimp = upf(s, h->geom_solimp, 5 * ng);
  m.geom_margin = upf(s, h->geom_margin, ng); m.geom_gap = upf(s, h->geom_gap, ng);
  m.pair_geom1 = upi(s, h->pair_geom1, m.npair); m.pair_geom2 = upi(s, h->pair_geom2, m.npair);
  { // packed broadphase record per pair: geoms + plane flag, and margin + bounding radii (plane pairs: of geom 2 only)
    std::vector<int> pi((size_t)std::max(m.npair, 1), 0); std::vector<float> rs(std::max(m.npair, 1), 0.0f);
    for (int k = 0; k < m.npair; k++) {
      int g1 = h->pair_geom1[k], g2 = h->pair_geom2[k]; bool plane = h->geom_type[g1] == FB_GEOM_PLANE;
      if (g1 >= 32768 || g2 >= 32768) { s->err = "too many geoms for the packed pair record"; return -3; }
      pi[k] = g1 | (g2 << 15) | (plane ? (1 << 30) : 0);
      double margin = std::max(h->geom_margin[g1], h->geom_margin[g2]);
      rs[k] = (float)(margin + h->geom_rbound[g2] + (plane ? 0.0 : h->geom_rbound[g1]));
    }
    m.pair_info = up(s, pi); m.pair_rsum = up(s, rs);
  }
  m.fluid_bodyid = upi(s, h->fluid_bodyid, m.nfluid); m.fluid_pos = upf3(s, h->fluid_pos, m.nfluid);
  m.fluid_quat = upf(s, h->fluid_quat, 4 * m.nfluid); m.fluid_size = upf3(s, h->fluid_size, m.nfluid); m.fluid_coef = upf(s, h->fluid_coef, 12 * m.nfluid);
  m.site_bodyid = upi(s, h->site_bodyid, m.nsite); m.site_type = upi(s, h->site_type, m.nsite);
  m.site_pos = upf3(s, h->site_pos, m.nsite); m.site_quat = upf(s, h->site_quat, 4 * m.nsite); m.site_size = upf3(s, h->site_size, m.nsite);
  m.tendon_adr = upi(s, h->tendon_adr, m.ntendon); m.tendon_num = upi(s, h->tendon_num, m.ntendon);
  m.wrap_dofid = upi(s, h->wrap_dofid, m.nwrap); m.wrap_qposadr = upi(s, h->wrap_qposadr, m.nwrap); m.wrap_coef = upf(s, h->wrap_coef, m.nwrap);
  int nu = m.nu;
  m.actuator_trntype = upi(s, h->actuator_trntype, nu); m.actuator_trnid = upi(s, h->actuator_trnid, nu); m.actuator_dyntype = upi(s, h->actuator_dyntype, nu);
  m.actuator_biastype = upi(s, h->actuator_biastype, nu); m.actuator_ctrllimited = upi(s, h->actuator_ctrllimited, nu);
  m.actuator_forcelimited = upi(s, h->actuator_forcelimited, nu); m.actuator_actadr = upi(s, h->actuator_actadr, nu);
  m.actuator_dynprm = upf(s, h->actuator_dynprm, 3 * nu); m.actuator_gainprm = upf(s, h->actuator_gainprm, 3 * nu); m.actuator_biasprm = upf(s, h->actuator_biasprm, 3 * nu);
  m.actuator_ctrlrange = upf(s, h->actuator_ctrlrange, 2 * nu); m.actuator_forcerange = upf(s, h->actuator_forcerange, 2 * nu);
  m.sensor_type = upi(s, h->sensor_type, m.nsensor); m.sensor_objid = upi(s, h->sensor_objid, m.nsensor);
  m.sensor_adr = upi(s, h->sensor_adr, m.nsensor); m.sensor_dim = upi(s, h->sensor_dim, m.nsensor);
  s->h_dof_parent.assign(h->dof_parentid, h->dof_parentid + nv); s->h_dof_Madr.assign(h->dof_Madr, h->dof_Madr + nv);
  s->h_qpos0.assign(h->qpos0, h->qpos0 + m.nq); s->h_body_parent.assign(h->body_parentid, h->body_parentid + m.nbody);
  s->h_jnt_type.assign(h->jnt_type, h->jnt_type + nj); s->h_jnt_qadr.assign(h->jnt_qposadr, h->jnt_qposadr + nj);
  s->h_jnt_dofadr.assign(h->jnt_dofadr, h->jnt_dofadr + nj); s->h_jnt_body.assign(h->jnt_bodyid, h->jnt_bodyid + nj);
  s->h_site_body.assign(h->site_bodyid, h->site_bodyid + m.nsite);
  return 0;
}

static int alloc_data(FbSim* s, int N) {
  DevData& d = s->d; const DevModel& m = s->m;
  memset(&d, 0, sizeof(d));
  d.N = N; d.Np = (N + FB_WPB - 1) / FB_WPB * FB_WPB; d.sens_mode = -1;
  // pass 1: lay the per-env record out (offsets in 4-byte slots); pass 2: one allocation, rebase the pointers
  std::vector<std::pair<void**, size_t>> fields;
  size_t off = 0;
#define FA(field, n) { off = (off + 3) & ~(size_t)3; fields.push_back({(void**)&d.field, off}); off += (size_t)(n); }   // arrays start on 16-byte boundaries
#define IA(field, n) FA(field, n)
  FA(qpos, m.nq) FA(qvel, m.nv) FA(act, m.na + 1) FA(ctrl, m.nu + 1) FA(qacc, m.nv) FA(dof_isd, m.nv) FA(time, 1)
  // vectors / matrices / inertias padded to whole float4s (fb_math.h: FB_V3S ...)
  FA(ref, 3) FA(xpos, FB_V3S * m.nbody) FA(xquat, 4 * m.nbody) FA(xmat, FB_M3S * m.nbody) FA(xipos, FB_V3S * m.nbody) FA(ximat, FB_M3S * m.nbody)
  FA(geom_xpos, FB_V3S * m.ngeom) FA(geom_xmat, FB_M3S * m.ngeom) FA(site_xpos, FB_V3S * (m.nsite + 1)) FA(site_xmat, FB_M3S * (m.nsite + 1))
  FA(Sang, FB_V3S * m.nv) FA(Slin, FB_V3S * m.nv) FA(inert10, FB_I10S * m.nbody) FA(crb10, FB_I10S * m.nbody)
  FA(qM, m.nM) FA(qLD, m.nM) FA(qLDe, m.nM)
  FA(bvel, FB_S6S * m.nbody) FA(bacc, FB_S6S * m.nbody) FA(bfrc, FB_S6S * m.nbody) FA(bfl, FB_S6S * m.nbody) FA(bfrc0, FB_S6S * m.nbody) FA(bdel, FB_S6S * m.nbody)
  FA(qfrc_bias, m.nv) FA(qfrc_passive, m.nv) FA(qfrc_actuator, m.nv) FA(qfrc_smooth, m.nv) FA(qfrc_zf, m.nv) FA(qfrc_constraint, m.nv) FA(qtmp, m.nv)
  FA(act_dot, m.na + 1) FA(actuator_force, m.nu + 1)
  IA(ncon, 1) FA(con_dist, FB_MAXCON) FA(con_pos, 3 * FB_MAXCON) FA(con_frame, 9 * FB_MAXCON) IA(con_geom1, FB_MAXCON) IA(con_geom2, FB_MAXCON)
  IA(con_efcadr, FB_MAXCON) IA(con_dim, FB_MAXCON) FA(con_mu, FB_MAXCON) FA(con_fric, 2 * FB_MAXCON)
  FA(tmp_con, 13 * 4 * FB_MAXCAND) IA(tmp_geom, 2 * 4 * FB_MAXCAND)
  IA(nefc, 1) IA(efc_type, FB_MAXEFC) IA(efc_id, FB_MAXEFC)
  FA(efc_pos, FB_MAXEFC) FA(efc_margin, FB_MAXEFC) FA(efc_D, FB_MAXEFC) FA(efc_R, FB_MAXEFC) FA(efc_K, FB_MAXEFC) FA(efc_B, FB_MAXEFC)
  FA(efc_imp, FB_MAXEFC) FA(efc_aref, FB_MAXEFC) FA(efc_b, FB_MAXEFC) FA(efc_force, FB_MAXEFC)
  IA(efc_la, FB_MAXEFC) IA(efc_lb, FB_MAXEFC) IA(efc_key, FB_MAXEFC) IA(prev_key, FB_MAXEFC) IA(prev_n, 1) FA(prev_lam, FB_MAXEFC)
  FA(sensordata, m.nsensordata + 1) FA(sensor_sum, m.nsensordata + 1) IA(flags, 1) IA(niter, 1) IA(hold, 1)
  // large, sparsely touched arrays last
  FA(efc_w, (size_t)S_NSLOT * FB_MAXEFC)
  FA(efc_A, (size_t)FB_MAXEFC * (FB_MAXEFC + 1) / 2) FA(efc_G, (size_t)FB_MAXEFC * (FB_MAXEFC + 1) / 2)
  FA(efc_J, (size_t)FB_MAXEFC * FB_JROW) FA(efc_Z, (size_t)FB_MAXEFC * FB_JROW)
#undef FA
#undef IA
  off = (off + 31) & ~(size_t)31;              // records start on 128-byte boundaries
  if ((double)off * d.Np >= 4.0e9) { s->err = "too many envs for 32-bit record indexing"; return -5; }
  d.rec = (unsigned)off;
  float* base = dalloc<float>(s, (size_t)d.Np * off);
  if (!base) { s->err = "out of device memory (env records)"; return -4; }
  for (auto& f : fields) *f.first = (void*)(base + f.second);
#ifdef FB_CLK
  d.clk = (long long*)dalloc<long long>(s, 32 * 4096);
#endif
  d.obs_dim = m.nq + m.nv + m.na + 2 * m.nsensordata + 12 + 3 * m.nsite + 3;
  d.obs = dalloc<float>(s, (size_t)d.obs_dim * d.Np);
  return 0;
}

// host <-> device transfers of one field: host side is AoS [N][n]; device side is n slots of every record
static void field_to_host(FbSim* s, const void* dev, int n, void* dst) {
  if (n <= 0) return;
  copy_rows_async(s, dst, (size_t)n * 4, dev, (size_t)s->d.rec * 4, (size_t)n * 4, s->d.N);
  sync_stream(s);
}
// padded device array (count elements of `width` floats every `stride` slots) -> compact host array [N][count * width]
static void field_to_host_strided(FbSim* s, const void* dev, int count, int width, int stride, float* dst) {
  std::vector<float> tmp((size_t)s->d.N * count * stride);
  field_to_host(s, dev, count * stride, tmp.data());
  for (int e = 0; e < s->d.N; e++) for (int i = 0; i < count; i++) for (int k = 0; k < width; k++)
    dst[((size_t)e * count + i) * width + k] = tmp[((size_t)e * count + i) * stride + k];
}
static void field_from_host(FbSim* s, void* dev, int n, const void* src) {
  if (n <= 0) return;
  copy_rows_async(s, dev, (size_t)s->d.rec * 4, src, (size_t)n * 4, (size_t)n * 4, s->d.N);
  for (int e = s->d.N; e < s->d.Np; e++) copy_async(s, (char*)dev + (size_t)e * s->d.rec * 4, src, (size_t)n * 4);   // pad envs mirror env 0
  sync_stream(s);
}
// device staging buffer for scatter-style uploads (ctrl, ghost pose, partial resets)
static int ensure_stage(FbSim* s, const char* who, size_t floats, size_t ints) {
  if (int rc = grow(s, who, s->stage_pool, floats, 4, "staging", "floats", [&](size_t r) { s->stage = dalloc<float>(s, r); })) return rc;
  return grow(s, who, s->stage_i_pool, ints, 4, "index staging", "ints", [&](size_t r) { s->stage_i = dalloc<int>(s, r); });
}

// The state bank's rows follow the handle's arrays: whatever replaces an observation / task program, the reference slots, the
// applied-force arrays or the parameter overlay drops the bank (the stream is idle: the callers synchronise first); fb_state_bank lays it out again.
static void state_drop(FbSim* s) {
  if (!s->st_bank) return;
  scope_free(s, s->st_scope);
  s->st_bank = nullptr; s->st_segs_dev = nullptr; s->st_slots = 0; s->st_written.clear(); s->st_stale = true;
}
// applied forces (FB_QFRC_APPLIED, FB_XFRC_APPLIED): compact device arrays [Np][n], both allocated zeroed on first use
static float* applied_ptr(FbSim* s, int field, int* n) {
  *n = field == FB_QFRC_APPLIED ? s->m.nv : 6 * s->m.nbody;
  return field == FB_QFRC_APPLIED ? s->d.qfrc_applied : s->d.xfrc_applied;
}
static int ensure_applied(FbSim* s) {
  if (s->d.qfrc_applied) return 0;
  if (sync_stream(s) != 0) return -2;
  state_drop(s);
  float *q, *x;
  if (int rc = scope_alloc(s, s->applied_scope, "out of device memory (applied forces)", [&] {
        q = dalloc<float>(s, (size_t)s->d.Np * s->m.nv); x = dalloc<float>(s, (size_t)s->d.Np * 6 * s->m.nbody); }))
    return rc;
  s->d.qfrc_applied = q; s->d.xfrc_applied = x;      // the step graph is captured again: DevData changed
  return 0;
}
// model-parameter overlay (fb_param_*): a row of every FbParam field in enum order, each segment on a 16-byte boundary; body_inertia
// takes four slots per body, as the model table the kernels read with 128-bit loads.  Last the env's M_damp [nM], derived from its
// dof_damping (the diagonal at dof_Madr), so that the damped factorisation reads it exactly as the compiled table
static int prm_slot(int p, int i) { return p == FB_P_BODY_INERTIA ? i + i / 3 : i; }
static void prm_layout(FbSim* s, const FbModel* h) {
  const int nb = h->nbody, nv = h->nv, nj = h->njnt, ng = h->ngeom, nu = h->nu;
  const int n[FB_NPARAMS] = {nb, 3 * nb, nv, nv, nj, 3 * ng, 3 * nu, 3 * nu, 3, 3, 1, 1};
  const double* src[FB_NPARAMS] = {h->body_mass, h->body_inertia, h->dof_armature, h->dof_damping, h->jnt_stiffness, h->geom_friction,
                                   h->actuator_gainprm, h->actuator_biasprm, h->opt_gravity, h->opt_wind, &h->opt_density, &h->opt_viscosity};
  unsigned off = 0;
  for (int p = 0; p < FB_NPARAMS; p++) {
    s->prm_n[p] = n[p]; s->d.prm_off[p] = (int)off;
    off += ((unsigned)(p == FB_P_BODY_INERTIA ? 4 * nb : n[p]) + 3) & ~3u;
  }
  s->d.prm_mdamp = (int)off; off += ((unsigned)h->nM + 3) & ~3u;
  s->d.prm_stride = off;
  s->h_prm0.assign(off, 0.0f);
  for (int p = 0; p < FB_NPARAMS; p++) for (int i = 0; i < n[p]; i++) s->h_prm0[s->d.prm_off[p] + prm_slot(p, i)] = (float)src[p][i];
  for (int i = 0; i < nv; i++) s->h_prm0[s->d.prm_mdamp + h->dof_Madr[i]] = (float)h->dof_damping[i];
}
static int ensure_prm(FbSim* s) {
  if (s->d.prm) return 0;
  if (sync_stream(s) != 0) return -2;
  state_drop(s);
  const size_t Np = s->d.Np, P = s->d.prm_stride;
  float *p, *lo, *hi; unsigned* cnt; DevPrmDraw* g;
  if (int rc = scope_alloc(s, s->prm_scope, "out of device memory (model parameters)", [&] {
        p = dalloc<float>(s, Np * P); cnt = dalloc<unsigned>(s, Np); lo = dalloc<float>(s, P); hi = dalloc<float>(s, P);
        g = (DevPrmDraw*)dalloc<unsigned char>(s, sizeof(DevPrmDraw)); }))
    return rc;
  std::vector<float> rows(Np * P);
  for (size_t e = 0; e < Np; e++) std::copy(s->h_prm0.begin(), s->h_prm0.end(), rows.begin() + e * P);
  if (copy_sync(s, p, rows.data(), sizeof(float) * rows.size()) != 0) return -2;
  s->prm_draw_host = DevPrmDraw{}; s->prm_draw_host.lo = lo; s->prm_draw_host.hi = hi;
  for (int k = 0; k < FB_NPARAMS; k++) s->prm_draw_host.n[k] = s->prm_n[k];
  s->prm_draw_dev = g; s->h_prm_lo = s->h_prm0; s->h_prm_hi = s->h_prm0;
  s->d.prm = p; s->d.prm_count = cnt; s->d.prm_draw = nullptr;      // (the counters start at 0; the step graph is captured again)
  return 0;
}
// values from outside, `rows` rows of the parameter: finite, non-negative where MuJoCo's field is, no stiffness on a joint without a spring
static bool prm_valid(FbSim* s, const char* who, int p, const float* v, size_t rows) {
  const bool nonneg = p != FB_P_ACTUATOR_GAINPRM && p != FB_P_ACTUATOR_BIASPRM && p != FB_P_GRAVITY && p != FB_P_WIND;
  const size_t k = (size_t)s->prm_n[p];
  for (size_t i = 0; i < rows * k; i++) {
    if (!std::isfinite(v[i])) { s->err = std::string(who) + ": non-finite value"; return false; }
    if (nonneg && v[i] < 0) { s->err = std::string(who) + ": negative value (mass, inertia, armature, damping, stiffness, friction, density and viscosity are >= 0)"; return false; }
    if (p == FB_P_JNT_STIFFNESS && v[i] != 0 && s->h_jnt_type[i % k] != FB_JNT_HINGE) {
      s->err = std::string(who) + ": joint " + std::to_string(i % k) + " is not a hinge: its stiffness must stay 0 (the step has springs on hinge joints only)"; return false; }
  }
  return true;
}

extern "C" {

const char* fb_version(void) { return kVersion; }

int fb_create(const FbModel* hm, int n_envs, int device, FbHandle* out) {
  if (!hm || !out || n_envs <= 0) return -1;
  FbSim* s = new FbSim();                  // (value-initialised: every field without an initialiser starts at zero)
  s->device = device; s->hm = *hm;
  if (dev_open(s, n_envs) != 0) { delete s; return -2; }
  int rc = build_model(s, hm);             // (every upload and allocation has completed when it returns)
  if (rc == 0) rc = alloc_data(s, n_envs);
  // nothing has been freed yet, so a missing entry is an upload or allocation that failed
  if (rc == 0 && std::count(s->allocs.begin(), s->allocs.end(), nullptr)) { s->err = "out of device memory (model and env data)"; rc = -4; }
  if (rc == 0) prm_layout(s, hm);
  *out = s;
  if (rc != 0) return rc;
  std::vector<float> q0((size_t)n_envs * hm->nq);
  for (int e = 0; e < n_envs; e++) for (int i = 0; i < hm->nq; i++) q0[(size_t)e * hm->nq + i] = (float)hm->qpos0[i];
  field_from_host(s, s->d.qpos, hm->nq, q0.data());
  return fb_forward(s);
}

int fb_destroy(FbHandle s) {
  if (!s) return -1;
  dev_close(s);
  for (void* p : s->allocs) dev_free(p);
  delete s;
  return 0;
}

#ifdef FB_CLK
extern "C" int fb_clk_read(FbHandle s, long long* dst) { if (!s) return -1; cudaStreamSynchronize(s->stream); cudaMemcpy(dst, s->d.clk, sizeof(long long) * 32 * 4096, cudaMemcpyDeviceToHost); return (int)(s->launches % 4096); }
#endif
#ifdef FB_EMU
// host-emulation build only (tests): one geom against a heightfield; out [max][7] = dist, pos[3], normal[3]; prism (may be null):
// per contact the triangle of the walk it came from (col_convex_hfield)
extern "C" int fb_emu_convex_hfield_prisms(int type, const float* gp, const float* gm, const float* gs, float margin, const float* hp, const float* hm,
                                           const float* hf_size, int nrow, int ncol, const float* data, float* out, int max, int* prism) {
  HfCon c[64]; M3 Gm, Hm; for (int k = 0; k < 9; k++) { Gm.m[k] = gm[k]; Hm.m[k] = hm[k]; }
  if (max > 64) max = 64;
  int n = col_convex_hfield(c, max, margin, type, v3(gp[0], gp[1], gp[2]), Gm, v3(gs[0], gs[1], gs[2]), v3(hp[0], hp[1], hp[2]), Hm, hf_size, nrow, ncol, data, prism);
  for (int k = 0; k < n; k++) { out[7 * k] = c[k].dist; out[7 * k + 1] = c[k].pos.x; out[7 * k + 2] = c[k].pos.y; out[7 * k + 3] = c[k].pos.z; out[7 * k + 4] = c[k].n.x; out[7 * k + 5] = c[k].n.y; out[7 * k + 6] = c[k].n.z; }
  return n;
}
extern "C" int fb_emu_convex_hfield(int type, const float* gp, const float* gm, const float* gs, float margin, const float* hp, const float* hm,
                                    const float* hf_size, int nrow, int ncol, const float* data, float* out /* [max][7] */, int max) {
  return fb_emu_convex_hfield_prisms(type, gp, gm, gs, margin, hp, hm, hf_size, nrow, ncol, data, out, max, nullptr);
}
extern "C" void fb_emu_convex_stats(long* out) { for (int i = 0; i < 4; i++) { out[i] = g_convex_stats[i]; g_convex_stats[i] = 0; } }
// host-emulation build only (tests): the fp32 generic-convex narrowphase on one pair; out = dist, pos[3], normal[3]
extern "C" int fb_emu_convex_pair(int t1, const float* p1, const float* m1, const float* s1, int t2, const float* p2, const float* m2, const float* s2,
                                  float margin, float* out) {
  M3 R1, R2; for (int k = 0; k < 9; k++) { R1.m[k] = m1[k]; R2.m[k] = m2[k]; }
  RawCon c; int n = col_convex(&c, margin, t1, v3(p1[0], p1[1], p1[2]), R1, v3(s1[0], s1[1], s1[2]), t2, v3(p2[0], p2[1], p2[2]), R2, v3(s2[0], s2[1], s2[2]));
  if (n) { out[0] = c.dist; out[1] = c.pos.x; out[2] = c.pos.y; out[3] = c.pos.z; out[4] = c.n.x; out[5] = c.n.y; out[6] = c.n.z; }
  return n;
}
// host-emulation build only (tests): one pair of any type the collision stage handles, through kcol_narrow's dispatch (a plane
// is t1 = FB_GEOM_PLANE with its normal the third column of m1; a generic pair the prefilter keeps then runs MPR as in kcol_mpr),
// then the contact frames as col_store makes them; out [4][13] = dist, pos[3], frame[9] per contact
struct PairGeoms { V3 s1, s2; M3 R1, R2; V3 size(int k) const { return k == 1 ? s1 : s2; } M3 rot(int k) const { return k == 1 ? R1 : R2; } };
extern "C" int fb_emu_pair(int t1, const float* p1, const float* m1, const float* s1, int t2, const float* p2, const float* m2, const float* s2,
                           float margin, float* out) {
  PairGeoms g; for (int k = 0; k < 9; k++) { g.R1.m[k] = m1[k]; g.R2.m[k] = m2[k]; }
  g.s1 = v3(s1[0], s1[1], s1[2]); g.s2 = v3(s2[0], s2[1], s2[2]);
  const V3 x1 = v3(p1[0], p1[1], p1[2]), x2 = v3(p2[0], p2[1], p2[2]);
  const bool plane = t1 == FB_GEOM_PLANE;
  RawCon rc[4];
  int n = col_narrow_pair(rc, margin, plane, t1, x1, t2, x2, plane ? col(g.R1, 2) : v3(0, 0, 0), g);
  if (n < 0) n = convex_mpr(rc, margin, t1, x1, g.R1, g.s1, t2, x2, g.R2, g.s2);
  for (int i = 0; i < n; i++) {
    V3 f1, f2; make_frame(rc[i].n, rc[i].t, f1, f2);
    float* o = out + 13 * i;
    o[0] = rc[i].dist; o[1] = rc[i].pos.x; o[2] = rc[i].pos.y; o[3] = rc[i].pos.z; o[4] = rc[i].n.x; o[5] = rc[i].n.y; o[6] = rc[i].n.z;
    o[7] = f1.x; o[8] = f1.y; o[9] = f1.z; o[10] = f2.x; o[11] = f2.y; o[12] = f2.z;
  }
  return n;
}
#endif
const char* fb_last_error(FbHandle s) { return s ? s->err.c_str() : "null handle"; }
int fb_n_envs(FbHandle s) { return s ? s->d.N : -1; }
int fb_n_envs_padded(FbHandle s) { return s ? s->d.Np : -1; }
int fb_record_stride(FbHandle s) { return s ? (int)s->d.rec : -1; }
long long fb_launch_count(FbHandle s) { return s ? s->launches : -1; }
int fb_sync(FbHandle s) { if (!s) return -1; return sync_stream(s); }
int fb_set_solver(FbHandle s, float tolerance, int max_iter) {
  if (!s) return -1;
  if (tolerance > 0) s->m.tolerance = tolerance;
  if (max_iter > 0) s->m.max_iter = max_iter;
  return 0;
}

int fb_forward(FbHandle s) {
  if (!s) return -1;
  dev_select(s);
  launch_step1(s);
  launch_step2(s, false);
  return sync_stream(s);
}

// the launch sequence of one control step: n x [ step2 ; step1 ], sensor accumulation restarted at the first substep
static void step_sequence(FbSim* s, int n_substeps) {
  for (int k = 0; k < n_substeps; k++) {
    launch_step2(s, true);
    s->d.sens_mode = (k == 0) ? 1 : 0;
    launch_step1(s);
    s->d.sens_mode = -1;
  }
  s->d.nsub_done = n_substeps;
  if (s->hold_pending) { fb_launch<ShNone, Ph<ph_clear_hold>>(s, K_MISC); s->hold_pending = 0; }
}
#ifndef FB_EMU
// Kernel parameters (DevModel, DevData by value) are frozen into a captured graph, so a graph is reused only while the
// parts of the handle state that the step kernels read are unchanged; staging pointers of scatter / reset launches are not
// read by them and are masked out of the comparison.
static DevData canonical(const DevData& d) {
  DevData c = d;
  c.sc_field = nullptr; c.sc_idx = nullptr; c.sc_vals = nullptr; c.sc_k = 0; c.sc_nan0 = 0; c.sc_stride = 0;
  c.rst_ids = nullptr; c.rst_qpos = nullptr; c.rst_qvel = nullptr; c.rst_n = 0; c.rst_has_qvel = 0; c.rst_hold = 0;
  return c;
}
// One control step, between the events fb_last_step_ms reads.  Its 7 n launches are replayed from a CUDA graph: captured the
// second time the same (n_substeps, hold) signature is stepped with unchanged handle state, so the first call still runs (and configures) plain launches.
static void step_run(FbSim* s, int n_substeps) {
  cudaEventRecord(s->ev0, s->stream);
  const int hold = s->hold_pending ? 1 : 0;
  bool done = false;
  if (s->graphs_on && !s->prof_on) {
    DevData c = canonical(s->d);
    FbSim::StepGraph& g = s->graph[hold];
    const bool same = g.seen && g.n_sub == n_substeps && memcmp(&c, &g.d, sizeof(DevData)) == 0 && memcmp(&s->m, &g.m, sizeof(DevModel)) == 0;
    if (same && g.exec) {
      if (cudaGraphLaunch(g.exec, s->stream) == cudaSuccess) {
        s->d.do_integrate = 1; s->d.sens_mode = -1; s->d.nsub_done = n_substeps; s->hold_pending = 0; s->launches += g.launches;
        done = true;
      } else { cudaGetLastError(); cudaGraphExecDestroy(g.exec); g.exec = nullptr; g.seen = false; }
    } else if (same && !g.failed) {
      long long l0 = s->launches; cudaGraph_t graph = nullptr;
      if (cudaStreamBeginCapture(s->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
        step_sequence(s, n_substeps);
        cudaError_t e1 = cudaStreamEndCapture(s->stream, &graph);
        if (e1 == cudaSuccess && graph && cudaGraphInstantiate(&g.exec, graph, 0) == cudaSuccess && cudaGraphLaunch(g.exec, s->stream) == cudaSuccess) {
          g.launches = s->launches - l0; done = true;
        } else { cudaGetLastError(); g.exec = nullptr; g.failed = true; s->launches = l0; s->hold_pending = hold; }
        if (graph) cudaGraphDestroy(graph);
      } else { cudaGetLastError(); g.failed = true; }
    } else {
      if (g.exec) { cudaGraphExecDestroy(g.exec); g.exec = nullptr; }
      g.seen = true; g.n_sub = n_substeps; g.d = c; g.m = s->m;
    }
  }
  if (!done) step_sequence(s, n_substeps);
  cudaEventRecord(s->ev1, s->stream);
}
static void graphs_drop(FbSim* s) {       // the launch sequence changed
  for (auto& g : s->graph) { if (g.exec) { cudaGraphExecDestroy(g.exec); g.exec = nullptr; } g.seen = false; }
}
float fb_last_step_ms(FbHandle s) {
  if (!s) return -1; float ms = 0; cudaEventSynchronize(s->ev1); cudaEventElapsedTime(&ms, s->ev0, s->ev1); return ms;
}
void* fb_stream(FbHandle s) { return s ? (void*)s->stream : nullptr; }
#else
static void step_run(FbSim* s, int n_substeps) { step_sequence(s, n_substeps); }
static void graphs_drop(FbSim*) {}
float fb_last_step_ms(FbHandle) { return 0; }
void* fb_stream(FbHandle) { return nullptr; }
#endif
int fb_step(FbHandle s, int n_substeps) {
  if (!s || n_substeps <= 0) return -1;
  dev_select(s);
  step_run(s, n_substeps);
  return launch_check(s, "fb_step");
}

static void* field_ptr(FbSim* s, int field, int* n) {
  const DevModel& m = s->m; DevData& d = s->d;
  switch (field) {
    case FB_QPOS: *n = m.nq; return d.qpos;
    case FB_QVEL: *n = m.nv; return d.qvel;
    case FB_ACT: *n = m.na; return d.act;
    case FB_CTRL: *n = m.nu; return d.ctrl;
    case FB_QACC: *n = m.nv; return d.qacc;
    case FB_QACC_WARMSTART: *n = m.nv; return d.qacc;        /* the dual solver warm-starts from forces; kept for ABI compatibility */
    case FB_SENSORDATA: *n = m.nsensordata; return d.sensordata;
    case FB_SENSOR_MEAN: *n = m.nsensordata; return d.sensor_sum;
    case FB_XPOS: *n = 3 * m.nbody; return d.xpos;            /* padded on the device (fb_math.h): host reads go through field_to_host_strided */
    case FB_XMAT: *n = 9 * m.nbody; return d.xmat;
    case FB_SITE_XPOS: *n = 3 * m.nsite; return d.site_xpos;
    case FB_SITE_XMAT: *n = 9 * m.nsite; return d.site_xmat;
    case FB_TIME: *n = 1; return d.time;
    case FB_QFRC_SMOOTH: *n = m.nv; return d.qfrc_smooth;
    case FB_QFRC_CONSTRAINT: *n = m.nv; return d.qfrc_constraint;
    case FB_QFRC_PASSIVE: *n = m.nv; return d.qfrc_passive;
    case FB_QFRC_BIAS: *n = m.nv; return d.qfrc_bias;
    case FB_QFRC_ACTUATOR: *n = m.nv; return d.qfrc_actuator;
    case FB_EFC_FORCE: *n = FB_MAXEFC; return d.efc_force;
    default: *n = -1; return nullptr;
  }
}

int fb_field_size(FbHandle s, int field) {
  if (!s) return -1;
  int n; if (field_ptr(s, field, &n)) return n;
  switch (field) {
    case FB_QFRC_APPLIED: return s->m.nv;
    case FB_XFRC_APPLIED: return 6 * s->m.nbody;
    case FB_SUBTREE_COM: return 3 * s->m.nbody;
    case FB_NCON: case FB_NEFC: case FB_SOLVER_NITER: case FB_FLAGS: return 1;
    case FB_QM_DENSE: return s->m.nv * s->m.nv;
    case FB_CONTACT: return 16 * FB_MAXCON;
    default: return -1;
  }
}

int fb_get(FbHandle s, int field, void* dst, int is_device) {
  if (!s || !dst) return -1;
  if (sync_stream(s) != 0) return -2;
  int n; void* p = field_ptr(s, field, &n);
  const DevModel& m = s->m; int N = s->d.N;
  if (field == FB_QFRC_APPLIED || field == FB_XFRC_APPLIED) {
    if (is_device) { s->err = "applied forces are compact [n_envs][n] arrays, not record fields: use fb_applied_ptrs"; return -1; }
    const float* a = applied_ptr(s, field, &n);
    if (a) return copy_sync(s, dst, a, sizeof(float) * (size_t)N * n);
    memset(dst, 0, sizeof(float) * (size_t)N * n);      // unset = zero
    return 0;
  }
  if (is_device) { if (!p) { s->err = "field has no device array"; return -1; } *(void**)dst = p; return 0; }
  float* out = (float*)dst;
  if (p) {
    if (field == FB_XPOS) field_to_host_strided(s, p, m.nbody, 3, FB_V3S, out);
    else if (field == FB_XMAT) field_to_host_strided(s, p, m.nbody, 9, FB_M3S, out);
    else if (field == FB_SITE_XPOS) field_to_host_strided(s, p, m.nsite, 3, FB_V3S, out);
    else if (field == FB_SITE_XMAT) field_to_host_strided(s, p, m.nsite, 9, FB_M3S, out);
    else field_to_host(s, p, n, out);
    if (field == FB_XPOS || field == FB_SITE_XPOS) {     // stored relative to ref
      std::vector<float> ref((size_t)3 * N); field_to_host(s, s->d.ref, 3, ref.data());
      for (int e = 0; e < N; e++) for (int i = 0; i < n; i++) out[(size_t)e * n + i] += ref[(size_t)e * 3 + i % 3];
    }
    if (field == FB_SENSOR_MEAN && s->d.nsub_done > 0) for (size_t i = 0; i < (size_t)N * n; i++) out[i] /= (float)s->d.nsub_done;
    return 0;
  }
  std::vector<int> iv(N);
  switch (field) {
    case FB_NCON: field_to_host(s, s->d.ncon, 1, iv.data()); for (int e = 0; e < N; e++) out[e] = (float)iv[e]; return 0;
    case FB_NEFC: field_to_host(s, s->d.nefc, 1, iv.data()); for (int e = 0; e < N; e++) out[e] = (float)iv[e]; return 0;
    case FB_SOLVER_NITER: field_to_host(s, s->d.niter, 1, iv.data()); for (int e = 0; e < N; e++) out[e] = (float)iv[e]; return 0;
    case FB_FLAGS: field_to_host(s, s->d.flags, 1, iv.data()); for (int e = 0; e < N; e++) out[e] = (float)iv[e]; return 0;
    case FB_SUBTREE_COM: {
      std::vector<float> crb((size_t)10 * m.nbody * N), ref((size_t)3 * N);
      field_to_host_strided(s, s->d.crb10, m.nbody, 10, FB_I10S, crb.data()); field_to_host(s, s->d.ref, 3, ref.data());
      for (int e = 0; e < N; e++) {
        float w[4] = {0, 0, 0, 0};         // the world's subtree (MuJoCo subtree_com[0]): the sum of its children's composite inertias
        for (int b = 1; b < m.nbody; b++) if (s->h_body_parent[b] == 0) for (int k = 0; k < 4; k++) w[k] += crb[((size_t)e * m.nbody + b) * 10 + k];
        for (int b = 0; b < m.nbody; b++) { const float* c = b ? &crb[((size_t)e * m.nbody + b) * 10] : w;
          for (int i = 0; i < 3; i++) out[((size_t)e * m.nbody + b) * 3 + i] = (c[0] > 0 ? c[1 + i] / c[0] : 0.0f) + ref[(size_t)e * 3 + i]; } }
      return 0; }
    case FB_QM_DENSE: {
      std::vector<float> qm((size_t)m.nM * N); field_to_host(s, s->d.qM, m.nM, qm.data());
      int nv = m.nv; memset(out, 0, sizeof(float) * (size_t)N * nv * nv);
      for (int e = 0; e < N; e++) for (int i = 0; i < nv; i++) { int t = 0; for (int j = i; j >= 0; j = s->h_dof_parent[j], t++) {
        float v = qm[(size_t)e * m.nM + s->h_dof_Madr[i] + t]; out[((size_t)e * nv + i) * nv + j] = v; out[((size_t)e * nv + j) * nv + i] = v; } }
      return 0; }
    case FB_CONTACT: {
      std::vector<float> dist((size_t)FB_MAXCON * N), pos((size_t)3 * FB_MAXCON * N), frame((size_t)9 * FB_MAXCON * N), mu((size_t)FB_MAXCON * N), ref((size_t)3 * N);
      std::vector<int> g1((size_t)FB_MAXCON * N), g2((size_t)FB_MAXCON * N), ea((size_t)FB_MAXCON * N), dm((size_t)FB_MAXCON * N), nc(N);
      field_to_host(s, s->d.con_dist, FB_MAXCON, dist.data()); field_to_host(s, s->d.con_pos, 3 * FB_MAXCON, pos.data());
      field_to_host(s, s->d.con_frame, 9 * FB_MAXCON, frame.data()); field_to_host(s, s->d.con_mu, FB_MAXCON, mu.data()); field_to_host(s, s->d.ref, 3, ref.data());
      field_to_host(s, s->d.con_geom1, FB_MAXCON, g1.data()); field_to_host(s, s->d.con_geom2, FB_MAXCON, g2.data());
      field_to_host(s, s->d.con_efcadr, FB_MAXCON, ea.data()); field_to_host(s, s->d.con_dim, FB_MAXCON, dm.data()); field_to_host(s, s->d.ncon, 1, nc.data());
      memset(out, 0, sizeof(float) * (size_t)N * 16 * FB_MAXCON);
      for (int e = 0; e < N; e++) for (int c = 0; c < nc[e] && c < FB_MAXCON; c++) {
        float* o = out + ((size_t)e * FB_MAXCON + c) * 16; size_t ec = (size_t)e * FB_MAXCON + c;
        o[0] = dist[ec];
        for (int i = 0; i < 3; i++) { o[1 + i] = pos[ec * 3 + i] + ref[(size_t)e * 3 + i]; o[4 + i] = frame[ec * 9 + i]; }
        o[7] = (float)g1[ec]; o[8] = (float)g2[ec]; o[9] = (float)dm[ec];
        o[12] = (float)ea[ec]; o[10] = o[12] >= 0 ? 1.0f : 0.0f; o[11] = mu[ec];
        for (int i = 0; i < 3; i++) o[13 + i] = frame[ec * 9 + 3 + i];
      }
      return 0; }
    default: s->err = "unknown field"; return -1;
  }
}

int fb_set(FbHandle s, int field, const float* src) {
  if (!s || !src) return -1;
  if (sync_stream(s) != 0) return -2;
  int n;
  if (field == FB_QFRC_APPLIED || field == FB_XFRC_APPLIED) {
    int rc = ensure_applied(s);
    if (rc != 0) return rc;
    float* a = applied_ptr(s, field, &n);
    return copy_sync(s, a, src, sizeof(float) * (size_t)s->d.N * n);      // (pad envs keep zero applied forces)
  }
  void* p = field_ptr(s, field, &n);
  if (!p || !(field == FB_QPOS || field == FB_QVEL || field == FB_ACT || field == FB_CTRL || field == FB_QACC_WARMSTART || field == FB_QACC || field == FB_TIME)) { s->err = "field is not writable"; return -1; }
  if (n > 0) field_from_host(s, p, n, src);
  return 0;
}

// scatter vals[N][k] (already on the device, row-major) into columns idx[k] (device ints, or NULL = 0..k-1) of `field`
static void launch_scatter(FbSim* s, float* field, const int* idx_dev, const float* vals_dev, int k, int nan_to_zero = 0, unsigned stride = 0) {
  s->d.sc_field = field; s->d.sc_idx = idx_dev; s->d.sc_vals = vals_dev; s->d.sc_k = k; s->d.sc_nan0 = nan_to_zero; s->d.sc_stride = stride;
  fb_launch<ShNone, Ph<ph_scatter>>(s, K_MISC);
  s->d.sc_stride = 0;
}

int fb_set_ctrl(FbHandle s, const float* ctrl, int is_device) {
  if (!s || !ctrl) return -1;
  const float* src = ctrl;
  const int k = s->act_map_dev ? s->n_action : s->m.nu;     // row length: actions (mapped on the device) or ctrl
  if (!is_device) {
    if (int rc = ensure_stage(s, "fb_set_ctrl", (size_t)s->d.N * std::max(k, s->m.nu), 0)) return rc;
    if (copy_async(s, s->stage, ctrl, sizeof(float) * (size_t)s->d.N * k) != 0) return -2;
    src = s->stage;
  }
  launch_scatter(s, s->d.ctrl, s->act_map_dev, src, k, s->act_map_dev ? 1 : 0);
  return launch_check(s, "fb_set_ctrl");
}
int fb_set_action_map(FbHandle s, const int32_t* ctrl_index, int n_action) {
  if (!s) return -1;
  const bool clear = !ctrl_index || n_action <= 0;      // back to plain ctrl rows
  for (int c = 0; !clear && c < n_action; c++) if (ctrl_index[c] >= s->m.nu || ctrl_index[c] < -1) { s->err = "fb_set_action_map: ctrl index out of range (valid: -1 = no target, 0..nu-1)"; return -1; }
  if (sync_stream(s) != 0) return -2;      // a scatter in flight may still read the old map
  scope_free(s, s->act_map_scope); s->act_map_dev = nullptr; s->n_action = 0;
  if (clear) return 0;
  std::vector<int> v(ctrl_index, ctrl_index + n_action);
  if (int rc = scope_alloc(s, s->act_map_scope, "fb_set_action_map: out of device memory", [&] { s->act_map_dev = up(s, v); })) { s->act_map_dev = nullptr; return rc; }
  s->n_action = n_action;
  return 0;
}

int fb_write_state(FbHandle s, int field, const int32_t* idx, int k, const float* vals) {
  if (!s || !idx || !vals || k <= 0) return -1;
  const bool applied = field == FB_QFRC_APPLIED || field == FB_XFRC_APPLIED;
  if (applied) { int rc = ensure_applied(s); if (rc != 0) return rc; }
  int n; float* p = applied ? applied_ptr(s, field, &n) : (float*)field_ptr(s, field, &n);
  if (!p || !(field == FB_QPOS || field == FB_QVEL || field == FB_ACT || applied)) {
    s->err = "fb_write_state: field must be qpos, qvel, act, qfrc_applied or xfrc_applied"; return -1; }
  for (int c = 0; c < k; c++) if (idx[c] < 0 || idx[c] >= n) { s->err = "fb_write_state: index out of range"; return -1; }
  // separate staging regions so that several writes can be in flight before the next sync
  size_t need = (size_t)s->d.N * s->m.nu + (size_t)4 * s->d.N * 16;
  if (k > 16) return -1;
  if (int rc = ensure_stage(s, "fb_write_state", need, 64)) return rc;
  int slot = s->ws_slot++ & 3;
  float* vdev = s->stage + (size_t)s->d.N * s->m.nu + (size_t)slot * s->d.N * 16;
  int* idev = s->stage_i + slot * 16;
  if (copy_async(s, idev, idx, sizeof(int) * k) != 0 || copy_async(s, vdev, vals, sizeof(float) * (size_t)s->d.N * k) != 0) return -2;
  launch_scatter(s, p, idev, vdev, k, 0, applied ? (unsigned)n : 0u);
  return launch_check(s, "fb_write_state");
}
int fb_applied_ptrs(FbHandle s, void** qfrc_dev, void** xfrc_dev) {
  if (!s) return -1;
  int rc = ensure_applied(s);
  if (rc != 0) return rc;
  if (qfrc_dev) *qfrc_dev = s->d.qfrc_applied;
  if (xfrc_dev) *xfrc_dev = s->d.xfrc_applied;
  return 0;
}
int fb_clear_applied(FbHandle s) {
  if (!s) return -1;
  if (!s->d.qfrc_applied) return 0;
  if (sync_stream(s) != 0) return -2;
  state_drop(s);
  scope_free(s, s->applied_scope);
  s->d.qfrc_applied = nullptr; s->d.xfrc_applied = nullptr;
  return 0;
}

int fb_param_size(FbHandle s, int p) { return (!s || p < 0 || p >= FB_NPARAMS) ? -1 : s->prm_n[p]; }
int fb_param_set(FbHandle s, int p, const int32_t* env_ids, int n, const float* vals, int) {
  if (!s) return -1;
  if (p < 0 || p >= FB_NPARAMS) { s->err = "fb_param_set: unknown parameter"; return -1; }
  if (!vals) { s->err = "fb_param_set: vals is NULL"; return -1; }
  const int N = s->d.N;
  if (!env_ids && n != N) { s->err = "fb_param_set: without env_ids, n must be n_envs"; return -1; }
  if (env_ids && n < 1) { s->err = "fb_param_set: n >= 1 envs"; return -1; }
  for (int k = 0; env_ids && k < n; k++) if (env_ids[k] < 0 || env_ids[k] >= N) { s->err = "fb_param_set: env id out of range"; return -1; }
  const size_t K = (size_t)s->prm_n[p];
  std::vector<float> v((size_t)n * K);
  if (copy_sync(s, v.data(), vals, sizeof(float) * v.size()) != 0) return -2;      // (host or device rows)
  if (!prm_valid(s, "fb_param_set", p, v.data(), n)) return -1;
  if (int rc = ensure_prm(s)) return rc;
  // read-modify-write of the parameter's segment of every env's row (dof_damping: and of the M_damp diagonal)
  const size_t P = s->d.prm_stride;
  auto write = [&](size_t off, size_t w, auto slot) {
    std::vector<float> rows((size_t)N * w);
    if (read_out(s, {{rows.data(), s->d.prm + off, P * 4, w * 4, (size_t)N}}) != 0) return -2;
    for (int k = 0; k < n; k++) {
      const size_t e = env_ids ? env_ids[k] : k;
      for (size_t i = 0; i < K; i++) rows[e * w + slot((int)i)] = v[k * K + i];
    }
    if (copy_rows_async(s, s->d.prm + off, P * 4, rows.data(), w * 4, w * 4, N) != 0) return -2;
    return sync_stream(s);
  };
  int rc = write(s->d.prm_off[p], p == FB_P_BODY_INERTIA ? 4 * K / 3 : K, [&](int i) { return prm_slot(p, i); });
  if (rc == 0 && p == FB_P_DOF_DAMPING) rc = write(s->d.prm_mdamp, s->m.nM, [&](int i) { return s->h_dof_Madr[i]; });
  return rc;
}
int fb_param_get(FbHandle s, int p, float* dst, int) {
  if (!s) return -1;
  if (p < 0 || p >= FB_NPARAMS) { s->err = "fb_param_get: unknown parameter"; return -1; }
  if (!dst) { s->err = "fb_param_get: dst is NULL"; return -1; }
  const int N = s->d.N;
  const size_t P = s->d.prm_stride, K = (size_t)s->prm_n[p], w = (size_t)(p == FB_P_BODY_INERTIA ? 4 * K / 3 : K);
  std::vector<float> rows((size_t)N * w), out((size_t)N * K);
  if (s->d.prm) { if (read_out(s, {{rows.data(), s->d.prm + s->d.prm_off[p], P * 4, w * 4, (size_t)N}}) != 0) return -2; }
  else for (int e = 0; e < N; e++) std::copy(s->h_prm0.begin() + s->d.prm_off[p], s->h_prm0.begin() + s->d.prm_off[p] + w, rows.begin() + (size_t)e * w);
  for (int e = 0; e < N; e++) for (size_t i = 0; i < K; i++) out[(size_t)e * K + i] = rows[(size_t)e * w + prm_slot(p, (int)i)];
  return copy_sync(s, dst, out.data(), sizeof(float) * out.size());      // (host or device memory)
}
int fb_param_draws(FbHandle s, int p, const float* lo, const float* hi, int shared, uint32_t seed) {
  if (!s) return -1;
  if (p < 0 || p >= FB_NPARAMS) { s->err = "fb_param_draws: unknown parameter"; return -1; }
  if (!lo != !hi) { s->err = "fb_param_draws: lo and hi are both given or both NULL"; return -1; }
  const int K = s->prm_n[p];
  if (lo) {
    if (!prm_valid(s, "fb_param_draws", p, lo, 1) || !prm_valid(s, "fb_param_draws", p, hi, 1)) return -1;
    for (int i = 0; i < K; i++) if (!(lo[i] <= hi[i])) { s->err = "fb_param_draws: lo > hi at element " + std::to_string(i); return -1; }
  } else if (!s->d.prm) return 0;          // nothing to stop
  if (int rc = ensure_prm(s)) return rc;
  DevPrmDraw& g = s->prm_draw_host;
  g.seed = seed; g.on[p] = lo ? 1 : 0; g.shared[p] = shared ? 1 : 0;
  for (int i = 0; lo && i < K; i++) { s->h_prm_lo[s->d.prm_off[p] + prm_slot(p, i)] = lo[i]; s->h_prm_hi[s->d.prm_off[p] + prm_slot(p, i)] = hi[i]; }
  const size_t bytes = sizeof(float) * s->d.prm_stride;
  if (copy_sync(s, (void*)g.lo, s->h_prm_lo.data(), bytes) != 0 || copy_sync(s, (void*)g.hi, s->h_prm_hi.data(), bytes) != 0 ||
      copy_sync(s, s->prm_draw_dev, &g, sizeof(g)) != 0) return -2;
  bool any = false;
  for (int k = 0; k < FB_NPARAMS; k++) any = any || g.on[k];
  s->d.prm_draw = any ? s->prm_draw_dev : nullptr;
  return 0;
}
int fb_param_clear(FbHandle s) {
  if (!s) return -1;
  if (!s->d.prm) return 0;
  if (sync_stream(s) != 0) return -2;
  state_drop(s);
  scope_free(s, s->prm_scope);
  s->d.prm = nullptr; s->d.prm_count = nullptr; s->d.prm_draw = nullptr; s->prm_draw_dev = nullptr;
  return 0;
}

static int do_reset(FbSim* s, const int32_t* env_ids, int n, const float* qpos, const float* qvel, int hold) {
  const DevModel& m = s->m; int N = s->d.N, Np = s->d.Np;
  if (sync_stream(s) != 0) return -2;
  std::vector<int> ids; std::vector<float> qp, qv;
  bool all = (env_ids == nullptr);
  if (all) n = N;
  for (int k = 0; k < n; k++) { int e = all ? k : env_ids[k]; if (e < 0 || e >= N) { s->err = "reset: env id out of range"; return -1; } ids.push_back(e); }
  qp.resize((size_t)ids.size() * m.nq);
  for (size_t k = 0; k < ids.size(); k++) for (int i = 0; i < m.nq; i++) qp[k * m.nq + i] = qpos ? qpos[k * m.nq + i] : (float)s->h_qpos0[i];
  if (qvel) qv.assign(qvel, qvel + (size_t)ids.size() * m.nv);
  if (all) for (int e = N; e < Np; e++) {          // pad envs mirror env 0
    ids.push_back(e); qp.insert(qp.end(), qp.begin(), qp.begin() + m.nq); if (qvel) qv.insert(qv.end(), qv.begin(), qv.begin() + m.nv);
  }
  int cnt = (int)ids.size();
  if (int rc = grow(s, "reset", s->rst_pool, std::max(cnt, Np), 4 * (1 + (size_t)m.nq + m.nv), "reset lists", "envs", [&](size_t r) {
        s->rst_ids_dev = dalloc<int>(s, r); s->rst_qpos_dev = dalloc<float>(s, r * m.nq); s->rst_qvel_dev = dalloc<float>(s, r * m.nv); }))
    return rc;
  const bool copied = copy_async(s, s->rst_ids_dev, ids.data(), sizeof(int) * cnt) == 0 && copy_async(s, s->rst_qpos_dev, qp.data(), sizeof(float) * qp.size()) == 0 &&
                      (!qvel || copy_async(s, s->rst_qvel_dev, qv.data(), sizeof(float) * qv.size()) == 0);
  if (sync_stream(s) != 0 || !copied) return -2;       // the host vectors go out of scope below
  s->d.rst_ids = s->rst_ids_dev; s->d.rst_qpos = s->rst_qpos_dev; s->d.rst_qvel = s->rst_qvel_dev; s->d.rst_n = cnt; s->d.rst_has_qvel = qvel ? 1 : 0; s->d.rst_hold = hold;
  fb_launch<ShNone, Ph<ph_reset_scatter>, Ph<ph_reset_draw>, Ph<ph_reset_count>>(s, K_MISC, 0, cnt);
  s->d.rst_n = 0;
  return 0;
}
int fb_reset(FbHandle s, const int32_t* env_ids, int n, const float* qpos, const float* qvel) {
  if (!s) return -1;
  int rc = do_reset(s, env_ids, n, qpos, qvel, 0);
  return rc != 0 ? rc : fb_forward(s);
}
int fb_reset_hold(FbHandle s, const int32_t* env_ids, int n, const float* qpos, const float* qvel) {
  if (!s || !env_ids || !qpos || n <= 0) return -1;
  int rc = do_reset(s, env_ids, n, qpos, qvel, 1);
  if (rc != 0) return rc;
  s->hold_pending = 1;
  return launch_check(s, "fb_reset_hold");
}

int fb_profile(FbHandle s, int enable) {
  if (!s) return -1;
  s->prof_on = enable ? 1 : 0;
  if (enable) { memset(s->prof_ms, 0, sizeof(s->prof_ms)); memset(s->prof_n, 0, sizeof(s->prof_n)); }
  return 0;
}
int fb_profile_read(FbHandle s, double* ms, long long* counts, int n) {
  if (!s || !ms || !counts) return -1;
  if (sync_stream(s) != 0) return -2;
  prof_collect(s);
  for (int k = 0; k < n && k < K_NKIND; k++) { ms[k] = s->prof_ms[k]; counts[k] = s->prof_n[k]; }
  return K_NKIND;
}
const char* fb_profile_name(int kind) { return (kind >= 0 && kind < K_NKIND) ? kKindNames[kind] : ""; }

// dynamic shared memory per CTA of the step kernel `kind` exactly as launch_step1 / launch_step2 request it (0: not a step kernel)
static size_t step_kernel_bytes(const FbSim* s, int kind) {
  const size_t blob = s->blob_in_smem ? (size_t)s->m.ts_blob_words * 4 : 0;
  switch (kind) {
    case K_SMOOTH: case K_FINISH: return slice_bytes(sizeof(ShTree), dyn_tsolve(s->m)) * FB_WPB + blob;
    case K_SOLVE: return sizeof(float) * FB_SOLVE_WARP_FLOATS * FB_SOLVE_WPB;
    case K_POS: return slice_bytes(sizeof(ShTree), dyn_pos(s->m)) * FB_WPB;
    case K_COL: return slice_bytes(sizeof(ShCol), dyn_col(s->m)) * FB_WPB;
    case K_PROJ: return slice_bytes(sizeof(ShCon), dyn_proj(s->m)) * FB_WPB;
    case K_VEL: return slice_bytes(sizeof(ShTree), dyn_vel(s->m)) * FB_WPB;
    default: return 0;
  }
}
int fb_step_kernel_smem(FbHandle s, int kind, int* bytes_per_cta, int* blocks_per_sm) {
  if (!s || !bytes_per_cta || !blocks_per_sm) return -1;
  const size_t bytes = (kind >= 0 && kind < K_NKIND) ? step_kernel_bytes(s, kind) : 0;
  if (bytes == 0) return -1;
  *bytes_per_cta = (int)bytes; *blocks_per_sm = 0;
  return step_kernel_blocks_per_sm(s, kind, bytes, blocks_per_sm);
}

int fb_obs_program(FbHandle s, const FbObsProgram* p) {
  if (!s || !p || p->n_items <= 0) return -1;
  if (sync_stream(s) != 0) return -2;
  const DevModel& m = s->m;
  int dim = 0; std::vector<int> offs;
  for (int i = 0; i < p->n_items; i++) {
    int k = p->kind[i], b = p->b[i];
    offs.push_back(dim);
    switch (k) {
      case FB_OBS_SENSOR_MEAN: case FB_OBS_SENSOR_NOW: case FB_OBS_ACT: case FB_OBS_QPOS: case FB_OBS_QVEL: case FB_OBS_TASK_TARGET: dim += b; break;
      case FB_OBS_SITES_EGO: case FB_OBS_REF_DISP: case FB_OBS_DOF_AXIS_EGO: dim += 3 * b; break;
      case FB_OBS_REF_QUAT: dim += 4 * b; break;
      case FB_OBS_ROOT_ZAXIS: case FB_OBS_SCALARS: case FB_OBS_SUBTREE_COM: dim += 3; break;
      case FB_OBS_ROOT_POSE: dim += 7; break;
      case FB_OBS_WORLD_CONTACT: dim += 1; break;
      default: s->err = "fb_obs_program: unknown item kind"; return -1;
    }
    if ((k == FB_OBS_REF_DISP || k == FB_OBS_REF_QUAT) && (!p->ref_qpos || p->ref_len <= 0)) { s->err = "fb_obs_program: reference table missing"; return -1; }
    if ((k == FB_OBS_QPOS || k == FB_OBS_QVEL || k == FB_OBS_SITES_EGO || k == FB_OBS_DOF_AXIS_EGO) && (p->a[i] < 0 || b < 0 || p->a[i] + b > p->n_list)) { s->err = "fb_obs_program: list range"; return -1; }
    if ((k == FB_OBS_SENSOR_MEAN || k == FB_OBS_SENSOR_NOW) && (p->a[i] < 0 || b < 0 || p->a[i] + b > m.nsensordata)) { s->err = "fb_obs_program: sensor range"; return -1; }
    if (k == FB_OBS_ACT && (p->a[i] < 0 || b < 0 || p->a[i] + b > m.na)) { s->err = "fb_obs_program: activation range"; return -1; }
    // (the kernels keep no composite inertia of the world body: its subtree CoM is only on the host, fb_get(FB_SUBTREE_COM))
    if (k == FB_OBS_SUBTREE_COM && (p->a[i] < 1 || p->a[i] >= m.nbody)) { s->err = "fb_obs_program: subtree_com body id (1 .. nbody - 1)"; return -1; }
    if ((k == FB_OBS_REF_DISP || k == FB_OBS_REF_QUAT) && b < 0) { s->err = "fb_obs_program: negative count"; return -1; }
  }
  for (int i = 0; i < p->n_items; i++) {          // entries of the index list, by the kind that reads them
    const int k = p->kind[i], lim = k == FB_OBS_QPOS ? m.nq : (k == FB_OBS_QVEL || k == FB_OBS_DOF_AXIS_EGO) ? m.nv : k == FB_OBS_SITES_EGO ? m.nsite : -1;
    if (lim < 0) continue;
    for (int j = 0; j < p->b[i]; j++) if (p->list[p->a[i] + j] < 0 || p->list[p->a[i] + j] >= lim) { s->err = "fb_obs_program: list entry out of range"; return -1; }
  }
  if (p->root_body <= 0 || p->root_body >= m.nbody) { s->err = "fb_obs_program: root body"; return -1; }
  // a replaced program's buffers are freed; the task program points into them (observation rows, per-env step inputs), so it goes too
  // and has to be uploaded again (fly_envs does: observation program, then task program)
  state_drop(s);
  scope_free(s, s->task_scope); s->d.task = nullptr;
  scope_free(s, s->obs_scope);
  std::vector<int> kind(p->kind, p->kind + p->n_items), a(p->a, p->a + p->n_items), b(p->b, p->b + p->n_items), list(p->list, p->list + std::max(p->n_list, 0));
  const int rc = scope_alloc(s, s->obs_scope, "out of device memory (observation program)", [&] {
    s->d.op_kind = up(s, kind); s->d.op_a = up(s, a); s->d.op_b = up(s, b); s->d.op_off = up(s, offs); s->d.op_list = up(s, list);
    if (p->ref_qpos && p->ref_len > 0) { std::vector<float> r(p->ref_qpos, p->ref_qpos + (size_t)7 * p->ref_len); s->d.op_ref = up(s, r); } else s->d.op_ref = nullptr;
    s->d.tobs = dalloc<float>(s, (size_t)dim * s->d.Np);
    s->op_step_dev = dalloc<int>(s, s->d.Np); s->op_first_dev = (unsigned char*)dalloc<int>(s, s->d.Np);
  });
  if (rc != 0) { s->d.tobs = nullptr; s->d.op_n = 0; return rc; }     // no program: the kernels skip the observation rows
  s->d.op_n = p->n_items; s->d.op_root_body = p->root_body; s->d.op_nsub = p->n_sub; s->d.op_ref_len = p->ref_len; s->d.op_ref_slot = 0;
  s->d.tobs_dim = dim; s->d.op_step = s->op_step_dev; s->d.op_first = s->op_first_dev;
  return dim;
}
int fb_ref_slots(FbHandle s, int slot_len) {
  if (!s || !s->d.tobs || slot_len <= 0) return -1;
  if (sync_stream(s) != 0) return -2;
  if (!s->ref_slots || s->ref_slot_len != slot_len || !s->d.op_ref_slot) state_drop(s);
  if (!s->ref_slots || s->ref_slot_len != slot_len) {          // (re)allocate: one [slot_len][7] table per env
    if (s->ref_slots && s->d.task && s->task_host.ref_bank) { scope_free(s, s->task_scope); s->d.task = nullptr; }      // it wrote into the old slots
    scope_free(s, s->ref_scope); s->ref_slots = nullptr; s->ref_slot_len = 0;
    if (int rc = scope_alloc(s, s->ref_scope, "out of device memory (reference slots)", [&] { s->ref_slots = dalloc<float>(s, (size_t)s->d.Np * 7 * slot_len); })) {
      s->ref_slots = nullptr; return rc; }
    s->ref_slot_len = slot_len;
  }
  s->d.op_ref = s->ref_slots; s->d.op_ref_len = slot_len; s->d.op_ref_slot = 1;
  return 0;
}
int fb_ref_slot_write(FbHandle s, const int32_t* env_ids, int n, const float* rows) {
  if (!s || !s->ref_slots || !s->d.op_ref_slot || !env_ids || !rows || n < 0) return -1;
  const size_t per = (size_t)7 * s->ref_slot_len;
  for (int k = 0; k < n; k++) {
    if (env_ids[k] < 0 || env_ids[k] >= s->d.N) { s->err = "fb_ref_slot_write: env id out of range"; return -1; }
    copy_async(s, s->ref_slots + per * env_ids[k], rows + per * k, sizeof(float) * per);
  }
  return sync_stream(s);                                        // the caller's rows may be reused right away
}
int fb_task_program(FbHandle s, const FbTaskProgram* p) {
  if (!s || !p) return -1;
  if (!s->d.tobs || !s->act_map_dev) { s->err = "fb_task_program: call fb_set_action_map and fb_obs_program first"; return -1; }
  const bool bank = (p->kind == FB_TASK_WALK || p->kind == FB_TASK_FLIGHT) && p->ref_bank;
  if (p->ref_bank && !bank) { s->err = "fb_task_program: ref_bank is for FB_TASK_WALK / FB_TASK_FLIGHT (walk_imitation / flight_imitation)"; return -1; }
  if (s->d.op_ref_slot && !bank) { s->err = "fb_task_program: per-env reference slots keep the host-side task code"; return -1; }
  if (bank) {
    if (!s->d.op_ref_slot || !s->ref_slots || s->ref_slot_len < 1) { s->err = "fb_task_program: ref_bank needs the per-env reference slots (fb_ref_slots) first"; return -1; }
    if (!s->rbank_dev) { s->err = "fb_task_program: ref_bank needs a trajectory bank (fb_ref_bank / fb_ref_bank_wide) first"; return -1; }
    if (p->n_pick <= 0 || !p->pick_traj) { s->err = "fb_task_program: ref_bank needs the trajectory indices to draw from (n_pick, pick_traj)"; return -1; }
    if (p->start_margin < 0 || p->max_episode_rows < 1 || p->future_steps < 0) { s->err = "fb_task_program: bad start_margin / max_episode_rows / future_steps"; return -1; }
    if (p->kind == FB_TASK_WALK && p->randomize_start) { s->err = "fb_task_program: walking starts every snippet at row 0 (randomize_start must be 0)"; return -1; }
    for (int k = 0; k < p->n_pick; k++) {
      const int j = p->pick_traj[k];
      if (j < 0 || j >= (int)s->rbank_len.size()) { s->err = "fb_task_program: trajectory index of pick_traj out of range of the bank"; return -1; }
      if (p->randomize_start && s->rbank_len[j] <= p->start_margin) {
        s->err = "fb_task_program: with randomize_start every trajectory to draw from must be longer than start_margin rows"; return -1; }
      if (p->kind == FB_TASK_WALK && s->rbank_len[j] <= p->future_steps + 1) {
        s->err = "fb_task_program: every walking trajectory to draw from must be longer than future_steps + 1 rows"; return -1; }
    }
    if (p->kind == FB_TASK_WALK) {          // the walking reward: the dataset's joints / sites in the bank rows and the walker's in the observation row
      const int nj = p->n_mocap_joints, ns = p->n_mocap_sites, dim = s->d.tobs_dim;
      if (nj <= 0 || ns < 0 || !p->mocap_qadr) { s->err = "fb_task_program: an FB_TASK_WALK ref_bank program needs the dataset's joints (n_mocap_joints, mocap_qadr)"; return -1; }
      for (int i = 0; i < nj; i++) if (p->mocap_qadr[i] < 0 || p->mocap_qadr[i] >= s->m.nq) { s->err = "fb_task_program: mocap_qadr entry out of range"; return -1; }
      if ((size_t)s->rbank_w != (size_t)FB_RBANK_W + 6 * (size_t)nj + 3 * (size_t)ns) {
        s->err = "fb_task_program: the bank rows are not 15 + 6 n_mocap_joints + 3 n_mocap_sites wide (fb_ref_bank_wide)"; return -1; }
      const int off[7] = {p->obs_root_pose_off, p->obs_root_qvel_off, p->obs_mocap_qpos_off, p->obs_mocap_qvel_off, p->obs_mocap_axes_off, p->obs_mocap_sites_off, p->obs_wing_qpos_off};
      const int wid[7] = {7, 6, nj, nj, 3 * nj, 3 * ns, p->n_wing};
      for (int k = 0; k < 7; k++) if (off[k] < 1 || off[k] + wid[k] > dim) {
        s->err = "fb_task_program: an FB_TASK_WALK ref_bank program needs the observation columns of the walker features (obs_*_off)"; return -1; }
      if (p->n_wing <= 0 || !p->wing_qadr || !p->wing_spring) { s->err = "fb_task_program: an FB_TASK_WALK ref_bank program needs the wing joints and their springs"; return -1; }
      for (int i = 0; i < p->n_wing; i++) if (p->wing_qadr[i] < 0 || p->wing_qadr[i] >= s->m.nq) { s->err = "fb_task_program: wing_qadr entry out of range"; return -1; }
      for (int k = 0; k < 4; k++) if (!(p->deep_mimic_std[k] > 0)) { s->err = "fb_task_program: deep_mimic_std must be positive"; return -1; }
      if (!(p->retract_margin > 0)) { s->err = "fb_task_program: retract_margin must be positive"; return -1; }
    }
  } else if (p->kind == FB_TASK_TEMPLATE || p->kind == FB_TASK_BALL) {
    if (p->ghost_qadr >= 0 || p->user_col >= 0 || p->n_noise > 0) { s->err = "fb_task_program: FB_TASK_TEMPLATE and FB_TASK_BALL (template_task, walk_on_ball) have no ghost, user action or reset noise"; return -1; }
    if (p->kind == FB_TASK_BALL && (p->ball_vadr < 0 || p->ball_vadr + 3 > s->m.nv || !(p->ball_margin > 0))) { s->err = "fb_task_program: FB_TASK_BALL needs the ball's dofs (ball_vadr) and a positive ball_margin"; return -1; }
  } else if (p->kind < FB_TASK_WALK || p->kind > FB_TASK_BALL) { s->err = "fb_task_program: unknown kind"; return -1;
  } else if (p->ref_len <= 0 || !p->ref_qpos || !p->ref_qvel) { s->err = "fb_task_program: reference / reset tables missing"; return -1; }
  if (!p->reset_qpos) { s->err = "fb_task_program: reference / reset tables missing"; return -1; }
  if (p->kind == FB_TASK_VISION && (!s->bank_dev || !s->hfield_dev || s->bank_n <= 0)) { s->err = "fb_task_program: FB_TASK_VISION needs fb_hfield_collision / fb_eye_program and fb_hfield_bank first"; return -1; }
  if ((p->kind == FB_TASK_FLIGHT || p->kind == FB_TASK_VISION) && (p->n_wing <= 0 || p->n_freq <= 0 || p->tab_len <= 0 || !p->wb_traj || !p->wb_phase || !p->wb_phase_mod || !p->wb_freqs || !p->wb_len)) { s->err = "fb_task_program: wing-beat tables missing"; return -1; }
  if (p->kind == FB_TASK_VISION && p->trench_cap > 0) {
    if (!p->trench_y || !p->trench_x || !p->trench_len) { s->err = "fb_task_program: trench centre lines missing"; return -1; }
    for (int k = 0; k < s->bank_n; k++) if (p->trench_len[k] < 2 || p->trench_len[k] > p->trench_cap || !(p->trench_x[2 * k + 1] > p->trench_x[2 * k])) { s->err = "fb_task_program: bad trench centre line"; return -1; }
  }
  if (sync_stream(s) != 0) return -2;
  const DevModel& m = s->m; const int Np = s->d.Np;
  state_drop(s);
  scope_free(s, s->task_scope); s->d.task = nullptr;
  DevTask t; memset(&t, 0, sizeof(t));
  t.kind = p->kind; t.root_qadr = p->root_qadr; t.root_vadr = p->root_vadr; t.ghost_qadr = p->ghost_qadr; t.ghost_vadr = p->ghost_vadr;
  t.root_body = s->d.op_root_body; t.user_col = p->user_col;
  for (int i = 0; i < 3; i++) { t.ghost_offset[i] = p->ghost_offset[i]; t.com_offset[i] = p->com_offset[i]; }
  t.dt = p->control_timestep; t.time_limit = p->time_limit; t.term_com = p->terminal_com_dist; t.term_linvel = p->terminal_linvel;
  t.term_angvel = p->terminal_angvel; t.term_qacc = p->terminal_qacc; t.term_height = p->terminal_height;
  t.velocimeter_adr = p->velocimeter_adr; t.gyro_adr = p->gyro_adr; t.com_body = p->com_body;
  t.ref_len = p->ref_len; t.obs_refdisp_off = p->obs_refdisp_off; t.obs_refquat_off = p->obs_refquat_off;
  float *ty = nullptr, *tx = nullptr; int* tl = nullptr; DevTask* dev = nullptr;
  const int rc = scope_alloc(s, s->task_scope, "out of device memory (task program)", [&] {
    auto upf32 = [&](const float* src, size_t n) { std::vector<float> v(src, src + n); return up(s, v); };
    auto upi32 = [&](const int32_t* src, size_t n) { std::vector<int> v(src, src + n); return up(s, v); };
    t.reset_qpos = upf32(p->reset_qpos, m.nq);
    if (p->kind == FB_TASK_BALL) { t.ball_vadr = p->ball_vadr; for (int i = 0; i < 3; i++) t.ball_target[i] = p->ball_target[i]; t.ball_margin = p->ball_margin; }
    if (!bank && p->kind != FB_TASK_TEMPLATE && p->kind != FB_TASK_BALL) { t.ref_qpos = upf32(p->ref_qpos, (size_t)7 * p->ref_len); t.ref_qvel = upf32(p->ref_qvel, (size_t)6 * p->ref_len); }
    else t.ref_len = 0;
    t.n_noise = p->noise_qadr ? p->n_noise : 0; t.noise_qadr = t.n_noise ? upi32(p->noise_qadr, t.n_noise) : nullptr; t.noise_amp = p->noise_amp; t.seed = p->seed;
    if (p->kind == FB_TASK_FLIGHT || p->kind == FB_TASK_VISION) {
      t.n_wing = p->n_wing; t.wing_qadr = upi32(p->wing_qadr, p->n_wing); t.wing_vadr = upi32(p->wing_vadr, p->n_wing); t.wing_ctrl = upi32(p->wing_ctrl, p->n_wing);
      t.n_freq = p->n_freq; t.tab_len = p->tab_len; const size_t nt = (size_t)p->n_freq * p->tab_len;
      t.wb_traj = upf32(p->wb_traj, nt * p->n_wing); t.wb_phase = upf32(p->wb_phase, nt); t.wb_phase_mod = upf32(p->wb_phase_mod, nt);
      t.wb_freqs = upf32(p->wb_freqs, p->n_freq); t.wb_len = upi32(p->wb_len, p->n_freq);
      t.wb_base_freq = p->wb_base_freq; t.wb_rel_range = p->wb_rel_range; t.wb_rate = p->wb_rate;
    }
    t.step = dalloc<int>(s, Np); t.needs_reset = dalloc<int>(s, Np); t.resetting = dalloc<int>(s, Np); t.episode = dalloc<int>(s, Np);
    t.wb_idx = dalloc<int>(s, Np); t.wb_pos = dalloc<int>(s, Np); t.has_uniform = dalloc<int>(s, Np);
    t.uniform = dalloc<float>(s, (size_t)8 * Np); t.wb_freq = dalloc<float>(s, Np); t.out = dalloc<float>(s, (size_t)4 * Np);
    t.ep_steps = dalloc<int>(s, Np);
    if (bank) {
      t.ref_bank = 1; t.rbank = s->rbank_dev; t.traj_off = s->rbank_off_dev; t.traj_len = s->rbank_len_dev; t.rbank_w = s->rbank_w;
      t.n_pick = p->n_pick; t.pick_traj = upi32(p->pick_traj, p->n_pick); t.randomize_start = p->randomize_start ? 1 : 0; t.start_margin = p->start_margin;
      t.max_episode_rows = p->max_episode_rows; t.future_steps = p->future_steps; t.slots = s->ref_slots; t.slot_len = s->ref_slot_len;
      t.ep_traj = dalloc<int>(s, Np); t.ep_start = dalloc<int>(s, Np); t.ep_row0 = dalloc<int>(s, Np); t.ep_n = dalloc<int>(s, Np); t.pin = dalloc<int>(s, (size_t)3 * Np);
      if (p->kind == FB_TASK_WALK) {
        t.n_mjnt = p->n_mocap_joints; t.n_msite = p->n_mocap_sites; t.mocap_qadr = upi32(p->mocap_qadr, p->n_mocap_joints);
        t.n_wing = p->n_wing; t.wing_qadr = upi32(p->wing_qadr, p->n_wing); t.wing_spring = upf32(p->wing_spring, p->n_wing);
        t.obs_root_pose_off = p->obs_root_pose_off; t.obs_root_qvel_off = p->obs_root_qvel_off; t.obs_mocap_qpos_off = p->obs_mocap_qpos_off;
        t.obs_mocap_qvel_off = p->obs_mocap_qvel_off; t.obs_mocap_axes_off = p->obs_mocap_axes_off; t.obs_mocap_sites_off = p->obs_mocap_sites_off;
        t.obs_wing_qpos_off = p->obs_wing_qpos_off;
        for (int k = 0; k < 4; k++) { t.dm_std[k] = p->deep_mimic_std[k]; t.dm_weight[k] = p->deep_mimic_weight[k]; }
        t.retract_margin = p->retract_margin;
        t.rw_part = dalloc<float>(s, (size_t)Np * FB_NY * 3);
      }
    }
    if (p->kind == FB_TASK_VISION) {
      for (int i = 0; i < 2; i++) { t.th_rng[i] = p->target_height_range[i]; t.ts_rng[i] = p->target_speed_range[i]; t.x_rng[i] = p->init_x_range[i]; t.y_rng[i] = p->init_y_range[i]; }
      for (int i = 0; i < 4; i++) t.hover_quat[i] = p->hover_quat[i];
      for (int i = 0; i < 3; i++) t.target_zaxis[i] = p->target_zaxis[i];
      t.fatal = p->floor_contacts_fatal;
      t.n_bank = s->bank_n; t.hf_nrow = s->hf_nrow; t.hf_ncol = s->hf_ncol; t.hf_ncm = s->hf_nbr * s->hf_nbc; t.hf_half = s->hf.size[0];
      t.bank = s->bank_dev; t.bank_hmax = s->bank_hmax_dev; t.bank_cmax = s->bank_cmax_dev; t.hf_data = s->hfield_dev; t.hf_hmax = s->hmax_dev; t.hf_cmax = s->cmax_dev;
      t.target = dalloc<float>(s, (size_t)2 * Np); t.pick = dalloc<int>(s, Np);
      t.trench_cap = 0; t.trench_x = t.trench_y = nullptr; t.trench_len = nullptr;
      if (p->trench_cap > 0) {
        ty = dalloc<float>(s, (size_t)p->trench_cap * s->bank_n); tx = dalloc<float>(s, (size_t)2 * s->bank_n); tl = dalloc<int>(s, s->bank_n);
        t.trench_cap = p->trench_cap; t.trench_x = tx; t.trench_y = ty; t.trench_len = tl;
      }
    }
    t.op_step = s->op_step_dev; t.op_first = s->op_first_dev;
    dev = (DevTask*)dalloc<unsigned char>(s, sizeof(DevTask));
  });
  if (rc != 0) return rc;
  std::vector<int> fill((size_t)Np);
  if (!bank) {          // (a dataset program's episode lengths are set per env by each reset)
    std::fill(fill.begin(), fill.end(), p->episode_steps); copy_sync(s, t.ep_steps, fill.data(), sizeof(int) * fill.size());
  }
  if (p->kind == FB_TASK_VISION) {
    std::fill(fill.begin(), fill.end(), -1); copy_sync(s, t.pick, fill.data(), sizeof(int) * fill.size());      // no terrain yet (a reset, or a loaded state row, copies one)
    if (t.trench_cap > 0) {
      copy_sync(s, ty, p->trench_y, sizeof(float) * (size_t)p->trench_cap * s->bank_n);
      copy_sync(s, tx, p->trench_x, sizeof(float) * 2 * s->bank_n);
      copy_sync(s, tl, p->trench_len, sizeof(int) * s->bank_n);
    }
  }
  copy_sync(s, dev, &t, sizeof(t));
  s->task_host = t; s->d.task = dev;
  return fb_task_reset_all(s);
}
int fb_task_reset_all(FbHandle s) {
  if (!s || !s->d.task) return -1;
  if (sync_stream(s) != 0) return -2;
  std::vector<int> ones((size_t)s->d.Np, 1);
  return copy_sync(s, s->task_host.needs_reset, ones.data(), sizeof(int) * ones.size());
}
int fb_task_set_reset_noise(FbHandle s, float amp) {
  if (!s || !s->d.task || !(amp >= 0)) return -1;
  if (sync_stream(s) != 0) return -2;
  s->task_host.noise_amp = amp;
  return copy_sync(s, (void*)s->d.task, &s->task_host, sizeof(DevTask));          // same pointers, new scalar
}
int fb_task_request_reset(FbHandle s, const int32_t* env_ids, int n) {
  if (!s || !s->d.task || (n > 0 && !env_ids) || n < 0) return -1;
  if (n == 0) return 0;
  if (sync_stream(s) != 0) return -2;
  const int one = 1;
  for (int k = 0; k < n; k++) {
    if (env_ids[k] < 0 || env_ids[k] >= s->d.N) { s->err = "fb_task_request_reset: env id out of range"; return -1; }
    copy_sync(s, s->task_host.needs_reset + env_ids[k], &one, sizeof(int));
  }
  return 0;
}
int fb_task_episodes(FbHandle s, int32_t* dst) {
  if (!s || !s->d.task || !dst) return -1;
  if (sync_stream(s) != 0) return -2;
  return copy_sync(s, dst, s->task_host.episode, sizeof(int) * (size_t)s->d.N);
}
int fb_task_uniforms(FbHandle s, const int32_t* env_ids, int n, const float* u) {
  if (!s || !s->d.task || !env_ids || !u || n < 0) return -1;
  if (sync_stream(s) != 0) return -2;
  const int one = 1;
  for (int k = 0; k < n; k++) {
    if (env_ids[k] < 0 || env_ids[k] >= s->d.N) { s->err = "fb_task_uniforms: env id out of range"; return -1; }
    copy_sync(s, s->task_host.uniform + (size_t)8 * env_ids[k], u + k, sizeof(float)); copy_sync(s, s->task_host.has_uniform + env_ids[k], &one, sizeof(int));
  }
  return 0;
}
int fb_task_uniform_rows(FbHandle s, const int32_t* env_ids, int n, const float* u) {
  if (!s || !s->d.task || !env_ids || !u || n < 0) return -1;
  if (sync_stream(s) != 0) return -2;
  const int one = 1;
  for (int k = 0; k < n; k++) {
    if (env_ids[k] < 0 || env_ids[k] >= s->d.N) { s->err = "fb_task_uniform_rows: env id out of range"; return -1; }
    copy_sync(s, s->task_host.uniform + (size_t)8 * env_ids[k], u + (size_t)8 * k, 8 * sizeof(float)); copy_sync(s, s->task_host.has_uniform + env_ids[k], &one, sizeof(int));
  }
  return 0;
}
// the highest point of one terrain, and of every block of FB_EYE_BLOCK x FB_EYE_BLOCK cells of it, border points included
// (the eye ray marcher's block maxima, fb_render.h)
static float terrain_maxima(const FbSim* s, const float* hk, float* cm) {
  const size_t cells = (size_t)s->hf_nrow * s->hf_ncol;
  float mx = hk[0]; for (size_t i = 1; i < cells; i++) mx = std::max(mx, hk[i]);
  for (int br = 0; br < s->hf_nbr; br++) for (int bc = 0; bc < s->hf_nbc; bc++) {
    float v = -3.0e38f;
    for (int iy = br * FB_EYE_BLOCK; iy <= std::min((br + 1) * FB_EYE_BLOCK, s->hf_nrow - 1); iy++)
      for (int ix = bc * FB_EYE_BLOCK; ix <= std::min((bc + 1) * FB_EYE_BLOCK, s->hf_ncol - 1); ix++) v = std::max(v, hk[(size_t)iy * s->hf_ncol + ix]);
    cm[(size_t)br * s->hf_nbc + bc] = v;
  }
  return mx;
}
int fb_hfield_bank(FbHandle s, int n_terrain, const float* heights) {
  if (!s || !s->hfield_dev || n_terrain <= 0 || !heights) { if (s) s->err = "fb_hfield_bank: set up the heightfield grid first (fb_hfield_collision / fb_eye_program)"; return -1; }
  if (sync_stream(s) != 0) return -2;
  const size_t cells = (size_t)s->hf_nrow * s->hf_ncol, ncm = (size_t)s->hf_nbr * s->hf_nbc;
  std::vector<float> hmax(n_terrain), cm(ncm * n_terrain);
  for (int k = 0; k < n_terrain; k++) hmax[k] = terrain_maxima(s, heights + cells * k, cm.data() + ncm * k);
  if (s->bank_dev && s->d.task && s->task_host.kind == FB_TASK_VISION) state_drop(s);
  if (s->bank_dev) {      // a replaced bank is freed; a vision task program pointing at it has to be uploaded again
    scope_free(s, s->bank_scope);
    if (s->d.task && s->task_host.kind == FB_TASK_VISION) { scope_free(s, s->task_scope); s->d.task = nullptr; }
  }
  if (int rc = scope_alloc(s, s->bank_scope, "out of device memory (terrain bank)", [&] {
        s->bank_dev = dalloc<float>(s, cells * n_terrain); s->bank_hmax_dev = dalloc<float>(s, n_terrain); s->bank_cmax_dev = dalloc<float>(s, ncm * n_terrain); })) {
    s->bank_dev = s->bank_hmax_dev = s->bank_cmax_dev = nullptr; s->bank_n = 0; return rc; }
  copy_sync(s, s->bank_dev, heights, sizeof(float) * cells * n_terrain); copy_sync(s, s->bank_hmax_dev, hmax.data(), sizeof(float) * n_terrain);
  copy_sync(s, s->bank_cmax_dev, cm.data(), sizeof(float) * cm.size());
  s->bank_n = n_terrain;
  return 0;
}
int fb_ref_bank(FbHandle s, int n_traj, const int32_t* traj_len, const float* rows) { return fb_ref_bank_wide(s, n_traj, traj_len, FB_RBANK_W, rows); }
int fb_ref_bank_wide(FbHandle s, int n_traj, const int32_t* traj_len, int row_width, const float* rows) {
  if (!s) return -1;
  if (n_traj <= 0 || !traj_len || !rows) { s->err = "fb_ref_bank: no trajectories"; return -1; }
  if (row_width < FB_RBANK_W) { s->err = "fb_ref_bank_wide: rows narrower than the 15 root columns"; return -1; }
  std::vector<int> off(n_traj), len(traj_len, traj_len + n_traj);
  size_t total = 0;
  for (int k = 0; k < n_traj; k++) {
    if (len[k] < 1) { s->err = "fb_ref_bank: empty trajectory"; return -1; }
    if (total > (size_t)INT32_MAX - (size_t)len[k]) { s->err = "fb_ref_bank: bank too large: more than 2^31 - 1 rows (int32 row index)"; return -1; }
    off[k] = (int)total; total += (size_t)len[k];
  }
  const size_t bytes = sizeof(float) * total * (size_t)row_width;      // (rows < 2^31, width < 2^31: no size_t overflow)
  if (bytes > dev_free_bytes()) { s->err = "fb_ref_bank: bank too large for the device's free memory"; return -4; }
  if (sync_stream(s) != 0) return -2;
  if (s->rbank_dev && s->d.task && s->task_host.ref_bank) state_drop(s);
  if (s->rbank_dev) {      // a replaced bank is freed; a dataset program drawing from it has to be uploaded again
    scope_free(s, s->rbank_scope);
    if (s->d.task && s->task_host.ref_bank) { scope_free(s, s->task_scope); s->d.task = nullptr; }
  }
  if (int rc = scope_alloc(s, s->rbank_scope, "out of device memory (trajectory bank)", [&] {
        s->rbank_dev = dalloc<float>(s, total * (size_t)row_width); s->rbank_off_dev = dalloc<int>(s, n_traj); s->rbank_len_dev = dalloc<int>(s, n_traj); })) {
    s->rbank_dev = nullptr; s->rbank_off_dev = s->rbank_len_dev = nullptr; s->rbank_len.clear(); s->rbank_w = 0; return rc; }
  copy_sync(s, s->rbank_dev, rows, bytes); copy_sync(s, s->rbank_off_dev, off.data(), sizeof(int) * n_traj); copy_sync(s, s->rbank_len_dev, len.data(), sizeof(int) * n_traj);
  s->rbank_len = len; s->rbank_w = row_width;
  return 0;
}
int fb_task_ref_pick(FbHandle s, const int32_t* env_ids, int n, const int32_t* traj, const int32_t* start) {
  if (!s || n < 0 || (n > 0 && (!env_ids || !traj || !start))) return -1;
  if (!s->d.task || !s->task_host.ref_bank) { s->err = "fb_task_ref_pick: needs a task program with ref_bank"; return -1; }
  std::vector<int> pins((size_t)3 * n);
  for (int k = 0; k < n; k++) {
    if (env_ids[k] < 0 || env_ids[k] >= s->d.N) { s->err = "fb_task_ref_pick: env id out of range"; return -1; }
    if (traj[k] < 0 || traj[k] >= (int)s->rbank_len.size()) { s->err = "fb_task_ref_pick: trajectory index out of range of the bank"; return -1; }
    if (start[k] < 0 || start[k] >= s->rbank_len[traj[k]]) { s->err = "fb_task_ref_pick: start step outside the trajectory"; return -1; }
    pins[3 * k] = 1; pins[3 * k + 1] = traj[k]; pins[3 * k + 2] = start[k];
  }
  if (sync_stream(s) != 0) return -2;
  for (int k = 0; k < n; k++) copy_async(s, s->task_host.pin + (size_t)3 * env_ids[k], pins.data() + 3 * k, 3 * sizeof(int));
  return sync_stream(s);                                        // `pins` goes out of scope
}
int fb_task_ref_state(FbHandle s, int32_t* traj, int32_t* start) {
  if (!s || !traj || !start) return -1;
  if (!s->d.task || !s->task_host.ref_bank) { s->err = "fb_task_ref_state: needs a task program with ref_bank"; return -1; }
  if (sync_stream(s) != 0) return -2;
  copy_async(s, traj, s->task_host.ep_traj, sizeof(int) * (size_t)s->d.N);
  copy_async(s, start, s->task_host.ep_start, sizeof(int) * (size_t)s->d.N);
  return sync_stream(s);
}
int fb_task_step(FbHandle s, const float* action, int is_device, int n_substeps) {
  if (!s || !s->d.task || !action || n_substeps <= 0) return -1;
  dev_select(s);
  fb_launch<ShNone, Ph<ph_task_reset>, Ph<ph_task_reset2>, Ph<ph_task_reset3>, Ph<ph_task_reset4>, Ph<ph_task_reset5>>(s, K_MISC, 0, s->d.N);      // envs whose last step was LAST
  int rc = fb_set_ctrl(s, action, is_device);                                           // action -> ctrl (NaN -> 0), staged rows stay readable
  if (rc != 0) return rc;
  fb_launch<ShNone, Ph<ph_task_before>, Ph<ph_task_commit>>(s, K_MISC, 0, s->d.N);
  s->hold_pending = 1;                                                                  // freshly reset envs are held through this step
  rc = fb_step(s, n_substeps);
  if (rc != 0) return rc;
  fb_launch<ShNone, Ph<ph_pack>, Ph<ph_task_reward>, Ph<ph_task_after>>(s, K_PACK, 0, s->d.N);
  return launch_check(s, "fb_task_step");
}
int fb_task_ptrs(FbHandle s, void** obs_dev, int* obs_dim, void** out_dev) {
  if (!s || !s->d.task) return -1;
  if (obs_dev) *obs_dev = s->d.tobs;
  if (obs_dim) *obs_dim = s->d.tobs_dim;
  if (out_dev) *out_dev = s->task_host.out;
  return 0;
}
int fb_task_read(FbHandle s, float* obs_host, float* out_host) {
  if (!s || !s->d.task) return -1;
  if (obs_host && copy_async(s, obs_host, s->d.tobs, sizeof(float) * (size_t)s->d.N * s->d.tobs_dim) != 0) return -2;
  if (out_host && copy_async(s, out_host, s->task_host.out, sizeof(float) * (size_t)4 * s->d.N) != 0) return -2;
  return sync_stream(s);
}
#ifndef FB_EMU
__global__ void __launch_bounds__(128) fb_render_kernel(DevData d, DevEye p) {
  const int e = blockIdx.x / p.n_cam, cam = blockIdx.x % p.n_cam;
  for (int px = threadIdx.x; px < p.size * p.size; px += blockDim.x) eye_pixel(d, p, e, cam, px / p.size, px % p.size);
}
static void launch_eyes(FbSim* s) {
  fb_render_kernel<<<s->d.N * s->eye.n_cam, 128, 0, s->stream>>>(s->d, s->eye);
  s->launches++;
}
#else
static void launch_eyes(FbSim* s) {
  emu_launch(s, "eye", 0, s->d.N, nullptr, [&](unsigned char*, int e) {
    for (int c = 0; c < s->eye.n_cam; c++) for (int px = 0; px < s->eye.size * s->eye.size; px++) eye_pixel(s->d, s->eye, e, c, px / s->eye.size, px % s->eye.size);
  });
}
#endif
// per-env heightfield buffer [Np][nrow * ncol] + highest point per env, shared by the collision and the eye cameras
static int ensure_hfield(FbSim* s, int nrow, int ncol) {
  if (s->hfield_dev) {
    if (s->hf_nrow != nrow || s->hf_ncol != ncol) { s->err = "heightfield grid differs from the one already allocated"; return -1; }
    return 0;
  }
  // block maxima for the eye ray marcher (fb_render.h: FB_EYE_BLOCK)
  const int nbr = (nrow - 1 + FB_EYE_BLOCK - 1) / FB_EYE_BLOCK, nbc = (ncol - 1 + FB_EYE_BLOCK - 1) / FB_EYE_BLOCK;
  if (int rc = scope_alloc(s, s->hf_scope, "out of device memory (heightfields)", [&] {
        s->hfield_dev = dalloc<float>(s, (size_t)nrow * ncol * s->d.Np); s->hmax_dev = dalloc<float>(s, s->d.Np);
        s->cmax_dev = dalloc<float>(s, (size_t)nbr * nbc * s->d.Np); })) {
    s->hfield_dev = s->hmax_dev = s->cmax_dev = nullptr; return rc; }
  s->hf_nrow = nrow; s->hf_ncol = ncol; s->hf_nbr = nbr; s->hf_nbc = nbc;
  return 0;
}
int fb_hfield_collision(FbHandle s, int geom, const float* size, int nrow, int ncol, const int32_t* pair_geom, int npair) {
  if (!s || !size || !pair_geom || npair <= 0 || npair > FB_MAXCAND || nrow < 2 || ncol < 2) return -1;
  if (geom < 0 || geom >= s->m.ngeom) { s->err = "fb_hfield_collision: geom id out of range"; return -1; }
  for (int k = 0; k < npair; k++) if (pair_geom[k] < 0 || pair_geom[k] >= s->m.ngeom) { s->err = "fb_hfield_collision: pair geom out of range"; return -1; }
  if (sync_stream(s) != 0) return -2;
  if (int rc = ensure_hfield(s, nrow, ncol)) return rc;
  graphs_drop(s);                          // a captured step graph holds the old DevHf and its pair list, which is freed here
  scope_free(s, s->hf_pair_scope); s->hf_on = false;
  DevHf& h = s->hf; h.geom = geom; h.nrow = nrow; h.ncol = ncol; h.npair = npair;
  for (int k = 0; k < 4; k++) h.size[k] = size[k];
  std::vector<int> pg(pair_geom, pair_geom + npair);
  if (int rc = scope_alloc(s, s->hf_pair_scope, "fb_hfield_collision: out of device memory", [&] { h.pair_geom = up(s, pg); })) return rc;
  h.data = s->hfield_dev; h.hmax = s->hmax_dev;
  s->hf_on = true;
  return 0;
}
int fb_eye_program(FbHandle s, const FbEyeProgram* p) {
  if (!s || !p) return -1;
  if (p->n_cam < 1 || p->n_cam > FB_MAXCAM || p->size < 1 || p->size > 512 || !(p->fovy_deg > 0 && p->fovy_deg < 180) || p->nrow < 0 || (p->nrow > 0 && (p->nrow < 2 || p->ncol < 2 || !(p->half_size > 0)))) { s->err = "fb_eye_program: bad camera / grid parameters"; return -1; }
  for (int c = 0; c < p->n_cam; c++) if (p->body[c] <= 0 || p->body[c] >= s->m.nbody) { s->err = "fb_eye_program: camera body out of range"; return -1; }
  if (sync_stream(s) != 0) return -2;
  scope_free(s, s->eye_scope); s->eye_out = nullptr;      // the images of the program this one replaces
  DevEye& y = s->eye; memset(&y, 0, sizeof(y));
  y.n_cam = p->n_cam; y.size = p->size; y.nrow = p->nrow; y.ncol = p->nrow > 0 ? p->ncol : 0;
  for (int c = 0; c < p->n_cam; c++) { y.body[c] = p->body[c]; for (int k = 0; k < 3; k++) y.pos[c][k] = p->pos[c][k]; for (int k = 0; k < 4; k++) y.quat[c][k] = p->quat[c][k]; }
  y.tan_half = tanf(0.5f * p->fovy_deg * 3.14159265358979f / 180.0f); y.half_size = p->half_size; y.z_offset = p->z_offset; y.zfar = p->zfar > 0 ? p->zfar : 50.0f;
  for (int k = 0; k < 3; k++) { y.sky_top[k] = p->sky_top[k]; y.sky_horizon[k] = p->sky_horizon[k]; y.ground[k] = p->ground[k]; }
  y.ambient = p->ambient; y.diffuse = p->diffuse;
  if (y.nrow > 0) if (int rc = ensure_hfield(s, y.nrow, y.ncol)) return rc;
  s->eye_bytes = (size_t)y.n_cam * y.size * y.size * 3;
  if (int rc = scope_alloc(s, s->eye_scope, "fb_eye_program: out of device memory (images)", [&] { s->eye_out = dalloc<unsigned char>(s, s->eye_bytes * s->d.Np); })) {
    s->eye_out = nullptr; return rc; }
  y.hfield = s->hfield_dev; y.hmax = s->hmax_dev; y.out = s->eye_out;
  y.cmax = (y.nrow > 0 && !getenv("FB_EYE_NO_SKIP")) ? s->cmax_dev : nullptr; y.nbr = s->hf_nbr; y.nbc = s->hf_nbc;
  return 0;
}
int fb_hfield_write(FbHandle s, const int32_t* env_ids, int n, const float* heights) {
  if (!s || !s->hfield_dev || !env_ids || !heights || n < 0) return -1;
  const size_t cells = (size_t)s->hf_nrow * s->hf_ncol;
  for (int k = 0; k < n; k++) {
    if (env_ids[k] < 0 || env_ids[k] >= s->d.N) { s->err = "fb_hfield_write: env id out of range"; return -1; }
    copy_async(s, s->hfield_dev + cells * env_ids[k], heights + cells * k, sizeof(float) * cells);
    std::vector<float> cm((size_t)s->hf_nbr * s->hf_nbc);
    const float mx = terrain_maxima(s, heights + cells * k, cm.data());
    if (sync_stream(s) != 0) return -2;
    copy_sync(s, s->cmax_dev + cm.size() * env_ids[k], cm.data(), sizeof(float) * cm.size());
    copy_sync(s, s->hmax_dev + env_ids[k], &mx, sizeof(float));
  }
  return 0;
}
int fb_render_eyes(FbHandle s) {
  if (!s || !s->eye_out) return -1;
  dev_select(s);
  launch_eyes(s);
  return launch_check(s, "fb_render_eyes");
}
int fb_eyes_ptr(FbHandle s, void** dev_ptr, int* bytes_per_env) {
  if (!s || !s->eye_out) return -1;
  if (dev_ptr) *dev_ptr = s->eye_out;
  if (bytes_per_env) *bytes_per_env = (int)s->eye_bytes;
  return 0;
}
int fb_eyes_read(FbHandle s, uint8_t* host_dst) {
  if (!s || !s->eye_out || !host_dst) return -1;
  return copy_sync(s, host_dst, s->eye_out, s->eye_bytes * s->d.N);
}
int fb_task_inputs(FbHandle s, const int32_t* step_idx, const uint8_t* first) {
  if (!s || !s->d.tobs || !step_idx || !first) return -1;
  if (copy_async(s, s->op_step_dev, step_idx, sizeof(int) * s->d.N) != 0) return -2;
  return copy_async(s, s->op_first_dev, first, s->d.N);
}
int fb_read_task_obs(FbHandle s, float* host_dst) {
  if (!s || !host_dst || !s->d.tobs) return -1;
  return copy_sync(s, host_dst, s->d.tobs, sizeof(float) * (size_t)s->d.N * s->d.tobs_dim);
}
int fb_pack_obs(FbHandle s) {
  if (!s) return -1;
  dev_select(s);
  fb_launch<ShNone, Ph<ph_pack>>(s, K_PACK);
  return launch_check(s, "fb_pack_obs");
}
int fb_read_obs(FbHandle s, float* host_dst) {
  if (!s || !host_dst) return -1;
  return copy_sync(s, host_dst, s->d.obs, sizeof(float) * (size_t)s->d.N * s->d.obs_dim);
}
int fb_obs_ptr(FbHandle s, void** dev_ptr, int* floats_per_env) {
  if (!s || !dev_ptr || !floats_per_env) return -1;
  *dev_ptr = s->d.obs; *floats_per_env = s->d.obs_dim;
  return 0;
}

}  // extern "C"

// ---- state rows (fb_state_*): the batched stand-in for physics.get_state() / physics.set_state()
// the row of the handle's current model, programs and applied-force arrays: segments in a fixed order, each on a 16-byte boundary
static std::vector<StSeg> state_layout(FbSim* s, unsigned* row, uint64_t* sig, int* hold_off) {
  const DevModel& m = s->m; const DevData& d = s->d;
  std::vector<StSeg> v; int off = 0; uint64_t h = 1469598103934665603ull;
  auto mix = [&](uint64_t x) { h = (h ^ x) * 1099511628211ull; };
  auto add = [&](int id, const void* base, unsigned stride, int n, int bytes = 0) {
    if (!base || n <= 0) return;
    StSeg g; g.base = const_cast<void*>(base); g.stride = stride; g.n = n; g.off = off; g.bytes = bytes;
    g.vec = (!bytes && stride % 4 == 0 && ((uintptr_t)base & 15) == 0) ? 1 : 0;
    v.push_back(g); mix((uint64_t)id); mix((uint64_t)n);
    off = (off + (bytes ? 1 : n) + 3) & ~3;
  };
  mix(1);                                    // layout version
  add(1, d.qpos, d.rec, m.nq); add(2, d.qvel, d.rec, m.nv); add(3, d.act, d.rec, m.na); add(4, d.ctrl, d.rec, m.nu); add(5, d.qacc, d.rec, m.nv);
  add(6, d.time, d.rec, 1); add(7, d.flags, d.rec, 1); add(8, d.niter, d.rec, 1);
  *hold_off = off; add(9, d.hold, d.rec, 1);
  add(10, d.prev_n, d.rec, 1); add(11, d.prev_key, d.rec, FB_MAXEFC); add(12, d.prev_lam, d.rec, FB_MAXEFC);
  add(13, d.sensordata, d.rec, m.nsensordata); add(14, d.sensor_sum, d.rec, m.nsensordata);
  add(15, d.obs, (unsigned)d.obs_dim, d.obs_dim);
  if (d.tobs) { add(16, d.tobs, (unsigned)d.tobs_dim, d.tobs_dim); add(17, s->op_step_dev, 1, 1); add(18, s->op_first_dev, 1, 1, 1); }
  if (d.op_ref_slot && s->ref_slots) add(19, s->ref_slots, (unsigned)(7 * s->ref_slot_len), 7 * s->ref_slot_len);
  if (d.qfrc_applied) { add(20, d.qfrc_applied, (unsigned)m.nv, m.nv); add(21, d.xfrc_applied, (unsigned)(6 * m.nbody), 6 * m.nbody); }
  if (d.prm) { add(22, d.prm, d.prm_stride, (int)d.prm_stride); add(23, d.prm_count, 1, 1); }
  mix(d.task ? (uint64_t)s->task_host.kind + 1 : 0); mix(d.task ? (uint64_t)s->task_host.ref_bank : 0);
  if (d.task) {
    const DevTask& t = s->task_host;
    add(30, t.step, 1, 1); add(31, t.needs_reset, 1, 1); add(32, t.resetting, 1, 1); add(33, t.episode, 1, 1); add(34, t.ep_steps, 1, 1);
    add(35, t.has_uniform, 1, 1); add(36, t.uniform, 8, 8); add(37, t.wb_idx, 1, 1); add(38, t.wb_pos, 1, 1); add(39, t.wb_freq, 1, 1);
    add(40, t.out, 4, 4);
    add(41, t.ep_traj, 1, 1); add(42, t.ep_start, 1, 1); add(43, t.ep_row0, 1, 1); add(44, t.ep_n, 1, 1); add(45, t.pin, 3, 3);
    add(46, t.target, 2, 2); add(47, t.pick, 1, 1);
  }
  *row = (unsigned)off; *sig = h;
  return v;
}
template <bool LOAD> struct StateWarp {
  StArgs a;
  FB_DEVM void operator()(unsigned char*, int w) const {
    int old_pick = -1;                       // a load: the env's terrain, read before any lane copies the row's over it
    if (LOAD) { WPAR_BEGIN old_pick = kstate_pick(a, w); WPAR_END }
    WPAR_BEGIN kstate_copy<LOAD>(a, w, lane); WPAR_END
    if (LOAD) { WPAR_BEGIN kstate_terrain(a, w, lane, old_pick); WPAR_END }
  }
};
// the (env, slot) pairs of the device lists env_ids / slots (NULL: the identity)
template <bool LOAD> static void launch_state(FbSim* s, const int* env_ids, const int* slots, int n) {
  warp_launch(s, "state", n, 0, StateWarp<LOAD>{{s->st_segs_dev, s->st_nseg, s->st_bank, s->st_row, env_ids, slots, n, s->d.task}});
}
static int state_ready(FbSim* s, const char* who) {
  if (s->st_bank) return 0;
  s->err = std::string(who) + (s->st_stale ? ": the state bank was dropped when the handle's programs, reference slots, applied-force arrays or parameter overlay changed: call fb_state_bank again"
                                           : ": no state bank (fb_state_bank)");
  return -1;
}
// the (env, slot) lists of a save / load on the device: envs at [0, n), slots at [n, 2n); a NULL list stays NULL (the identity)
static int state_ids(FbSim* s, const int32_t* env_ids, const int32_t* slots, int n, const int** env_dev, const int** slot_dev) {
  *env_dev = *slot_dev = nullptr;
  if (int rc = grow(s, "state bank", s->st_ids_pool, 2 * (size_t)std::max(n, s->d.Np), 4, "env and slot lists", "2 envs", [&](size_t r) {
        s->st_ids_dev = dalloc<int>(s, r); })) return rc;
  if (env_ids) { if (copy_async(s, s->st_ids_dev, env_ids, sizeof(int) * n) != 0) return -2; *env_dev = s->st_ids_dev; }
  if (slots) { if (copy_async(s, s->st_ids_dev + n, slots, sizeof(int) * n) != 0) return -2; *slot_dev = s->st_ids_dev + n; }
  return 0;
}
extern "C" {

int fb_state_slots(FbHandle s) {
  if (!s) return -1;
  unsigned row; uint64_t sig; int ho; state_layout(s, &row, &sig, &ho);
  return (int)row;
}
uint64_t fb_state_signature(FbHandle s) {
  if (!s) return 0;
  unsigned row; uint64_t sig; int ho; state_layout(s, &row, &sig, &ho);
  return sig;
}
int fb_state_bank(FbHandle s, int n_slots) {
  if (!s || n_slots < 0) return -1;
  if (sync_stream(s) != 0) return -2;
  state_drop(s); s->st_stale = false;
  if (n_slots == 0) return 0;
  unsigned row; uint64_t sig; int ho;
  std::vector<StSeg> segs = state_layout(s, &row, &sig, &ho);
  const size_t bytes = (size_t)n_slots * row * 4;
  if (bytes > dev_free_bytes()) { s->err = "fb_state_bank: the bank does not fit the device's free memory"; return -4; }
  if (int rc = scope_alloc(s, s->st_scope, "fb_state_bank: out of memory", [&] {
        s->st_bank = dalloc<unsigned>(s, (size_t)n_slots * row); s->st_segs_dev = (StSeg*)dalloc<unsigned char>(s, sizeof(StSeg) * segs.size()); })) {
    s->st_bank = nullptr; s->st_segs_dev = nullptr; return rc; }
  copy_sync(s, s->st_segs_dev, segs.data(), sizeof(StSeg) * segs.size());
  s->st_nseg = (int)segs.size(); s->st_row = row; s->st_sig = sig; s->st_hold_off = ho; s->st_slots = n_slots; s->st_written.assign(n_slots, 0);
  return 0;
}
int fb_state_save(FbHandle s, const int32_t* env_ids, const int32_t* slots, int n) {
  if (!s) return -1;
  if (state_ready(s, "fb_state_save") != 0) return -1;
  if (!env_ids && !slots) n = s->d.N;
  if (n <= 0) return n == 0 ? 0 : -1;
  std::vector<char> seen(s->st_slots, 0);
  for (int k = 0; k < n; k++) {
    const int e = env_ids ? env_ids[k] : k, sl = slots ? slots[k] : k;
    if (e < 0 || e >= s->d.N) { s->err = "fb_state_save: env id out of range"; return -1; }
    if (sl < 0 || sl >= s->st_slots) { s->err = "fb_state_save: slot out of range of the bank"; return -1; }
    if (seen[sl]) { s->err = "fb_state_save: a slot may be written once per call"; return -1; }
    seen[sl] = 1;
  }
  dev_select(s);
  const int *ed, *sd; int rc = state_ids(s, env_ids, slots, n, &ed, &sd);
  if (rc != 0) return rc;
  launch_state<false>(s, ed, sd, n);
  for (int k = 0; k < n; k++) s->st_written[slots ? slots[k] : k] = s->hold_pending ? 2 : 1;
  return launch_check(s, "fb_state_save");
}
int fb_state_load(FbHandle s, const int32_t* slots, const int32_t* env_ids, int n) {
  if (!s) return -1;
  if (state_ready(s, "fb_state_load") != 0) return -1;
  if (!env_ids && !slots) n = s->d.N;
  if (n <= 0) return n == 0 ? 0 : -1;
  std::vector<char> seen(s->d.N, 0); bool held = false;
  for (int k = 0; k < n; k++) {
    const int e = env_ids ? env_ids[k] : k, sl = slots ? slots[k] : k;
    if (e < 0 || e >= s->d.N) { s->err = "fb_state_load: env id out of range"; return -1; }
    if (sl < 0 || sl >= s->st_slots) { s->err = "fb_state_load: slot out of range of the bank"; return -1; }
    if (!s->st_written[sl]) { s->err = "fb_state_load: slot " + std::to_string(sl) + " was never written"; return -1; }
    if (seen[e]) { s->err = "fb_state_load: env " + std::to_string(e) + " appears twice"; return -1; }
    seen[e] = 1; held = held || s->st_written[sl] == 2;
  }
  dev_select(s);
  const int *ed, *sd; int rc = state_ids(s, env_ids, slots, n, &ed, &sd);
  if (rc != 0) return rc;
  launch_state<true>(s, ed, sd, n);
  // what the row does not carry is a function of it: the position / velocity stage, for the loaded envs (all of them: the step's own launches)
  if (n == s->d.N) launch_step1(s); else launch_step1_ids(s, ed, n);
  if (held) s->hold_pending = 1;             // a restored env waits for its reset: the next step holds it and clears the hold
  return launch_check(s, "fb_state_load");
}
int fb_state_read(FbHandle s, const int32_t* slots, int n, void* host_dst) {
  if (!s || !host_dst || n < 0) return -1;
  if (state_ready(s, "fb_state_read") != 0) return -1;
  for (int k = 0; k < n; k++) {
    const int sl = slots ? slots[k] : k;
    if (sl < 0 || sl >= s->st_slots) { s->err = "fb_state_read: slot out of range of the bank"; return -1; }
    if (!s->st_written[sl]) { s->err = "fb_state_read: slot " + std::to_string(sl) + " was never written"; return -1; }
  }
  if (sync_stream(s) != 0) return -2;
  const size_t rb = (size_t)s->st_row * 4;
  if (!slots) return copy_sync(s, host_dst, s->st_bank, rb * n);
  for (int k = 0; k < n; k++) copy_sync(s, (char*)host_dst + rb * k, s->st_bank + (size_t)s->st_row * slots[k], rb);
  return 0;
}
int fb_state_substeps(FbHandle s, int n_substeps) {
  if (!s) return -1;
  if (n_substeps > 0) s->d.nsub_done = n_substeps;
  return s->d.nsub_done;
}
int fb_state_write(FbHandle s, const int32_t* slots, int n, const void* host_src) {
  if (!s || !host_src || n < 0) return -1;
  if (state_ready(s, "fb_state_write") != 0) return -1;
  for (int k = 0; k < n; k++) { const int sl = slots ? slots[k] : k; if (sl < 0 || sl >= s->st_slots) { s->err = "fb_state_write: slot out of range of the bank"; return -1; } }
  if (sync_stream(s) != 0) return -2;
  const size_t rb = (size_t)s->st_row * 4;
  for (int k = 0; k < n; k++) {
    const int sl = slots ? slots[k] : k;
    const unsigned* src = (const unsigned*)((const char*)host_src + rb * k);
    copy_sync(s, s->st_bank + (size_t)s->st_row * sl, src, rb);
    s->st_written[sl] = src[s->st_hold_off] ? 2 : 1;
  }
  return 0;
}

}  // extern "C"

// -------------------------------------------------------------------------------------------
// inverse kinematics (fb_ik_*; fb_ik.h): its own kernel parameter (DevIk) and buffers (ik_scope), bounded launches
#define FB_IK_LAUNCH_ITERS (4 * FB_IK_CHECK)       // iterations per launch: the host reads the live count once per launch
struct IkWarp {
  DevModel m; DevData d; DevIk p;
  FB_DEVM void operator()(unsigned char* sh, int e) const { kik_run(m, d, p, reinterpret_cast<float*>(sh), e); }
};
// one bounded launch; *live: the problems still iterating after it
static int ik_launch(FbSim* s, int* live) {
  static const int zero = 0;
  if (copy_async(s, s->ik.live, &zero, sizeof(int)) != 0) return -2;
  warp_launch(s, "ik", s->ik.n, sizeof(float) * FB_IK_SH(s->ik.n_fdof), IkWarp{s->m, s->d, s->ik});
  if (launch_check(s, "fb_ik_solve") != 0 || copy_async(s, live, s->ik.live, sizeof(int)) != 0) return -2;
  return sync_stream(s);
}

extern "C" {

int fb_ik_program(FbHandle s, const FbIkProgram* p) {
  if (!s || !p) return -1;
  const DevModel& m = s->m;
  if (p->n_sites < 1 || p->n_sites > FB_IK_MAXSITE || !p->site_ids) { s->err = "fb_ik_program: 1 .. 64 sites"; return -1; }
  if (p->n_jnts < 1 || !p->jnt_ids) { s->err = "fb_ik_program: no joints to fit"; return -1; }
  for (int k = 0; k < p->n_sites; k++) if (p->site_ids[k] < 0 || p->site_ids[k] >= m.nsite) { s->err = "fb_ik_program: site id out of range"; return -1; }
  std::vector<char> seen(m.njnt, 0);
  for (int k = 0; k < p->n_jnts; k++) {
    const int j = p->jnt_ids[k];
    if (j < 0 || j >= m.njnt) { s->err = "fb_ik_program: joint id out of range"; return -1; }
    if (seen[j]++) { s->err = "fb_ik_program: joint listed twice"; return -1; }
    if (s->h_jnt_type[j] != FB_JNT_HINGE && s->h_jnt_type[j] != FB_JNT_FREE) { s->err = "fb_ik_program: only hinge and free joints can be fitted (ball joints cannot)"; return -1; }
  }
  if (!(std::isfinite(p->reg_strength) && std::isfinite(p->lr) && std::isfinite(p->beta) && std::isfinite(p->progress_threshold)) || p->max_steps < 1) {
    s->err = "fb_ik_program: non-finite parameter or max_steps < 1"; return -1;
  }
  if (sync_stream(s) != 0) return -2;
  // fitted dofs in joint order; the sites below each (site body at or under the dof's body)
  std::vector<int> fdof, hq, jt, jq, jf; std::vector<unsigned long long> below;
  for (int k = 0; k < p->n_jnts; k++) {
    const int j = p->jnt_ids[k], t = s->h_jnt_type[j], nd = t == FB_JNT_FREE ? 6 : 1, b = s->h_jnt_body[j];
    jt.push_back(t); jq.push_back(s->h_jnt_qadr[j]); jf.push_back((int)fdof.size());
    unsigned long long mask = 0;
    for (int q = 0; q < p->n_sites; q++) for (int a = s->h_site_body[p->site_ids[q]]; a > 0; a = s->h_body_parent[a]) if (a == b) { mask |= 1ull << q; break; }
    for (int i = 0; i < nd; i++) { fdof.push_back(s->h_jnt_dofadr[j] + i); hq.push_back(t == FB_JNT_HINGE ? s->h_jnt_qadr[j] : -1); below.push_back(mask); }
  }
  std::vector<unsigned char> inc(3 * p->n_sites, 1);
  if (p->include) for (int k = 0; k < 3 * p->n_sites; k++) inc[k] = p->include[k] ? 1 : 0;
  std::vector<int> sid(p->site_ids, p->site_ids + p->n_sites);
  scope_free(s, s->ik_scope);
  const int Np = s->d.Np, nfd = (int)fdof.size();
  DevIk& k = s->ik; k = DevIk{};
  k.n_site = p->n_sites; k.n_fdof = nfd; k.n_fjnt = p->n_jnts; k.iters = FB_IK_LAUNCH_ITERS; k.max_steps = p->max_steps;
  k.reg = p->reg_strength; k.lr = p->lr; k.beta = p->beta; k.thr = p->progress_threshold;
  if (int rc = scope_alloc(s, s->ik_scope, "out of device memory (IK program)", [&] {
        k.site_id = up(s, sid); k.include = up(s, inc); k.fdof = up(s, fdof); k.fdof_hqadr = up(s, hq); k.below = up(s, below);
        k.fjnt_type = up(s, jt); k.fjnt_qadr = up(s, jq); k.fjnt_fd0 = up(s, jf);
        k.target = dalloc<float>(s, (size_t)Np * 3 * p->n_sites); k.u = dalloc<float>(s, (size_t)Np * nfd);
        k.step = dalloc<int>(s, Np); k.done = dalloc<int>(s, Np); k.err = dalloc<float>(s, Np); k.err_first = dalloc<float>(s, Np);
        k.steps = dalloc<int>(s, Np); k.success = dalloc<unsigned char>(s, Np); k.live = dalloc<int>(s, 1); })) {
    s->ik = DevIk{}; return rc; }
  s->ik_solved = 0;
  return 0;
}

int fb_ik_solve(FbHandle s, int n, const float* target_xpos, const float* init_qpos) {
  if (!s) return -1;
  DevIk& p = s->ik;
  if (!p.live) { s->err = "fb_ik_solve: no IK program (fb_ik_program)"; return -1; }
  if (n < 1 || n > s->d.N || !target_xpos) { s->err = "fb_ik_solve: 1 <= n <= n_envs problems with targets"; return -1; }
  const int nq = s->m.nq, nt = 3 * p.n_site;
  for (size_t i = 0; i < (size_t)n * nt; i++) if (std::isinf(target_xpos[i])) { s->err = "fb_ik_solve: infinite target component"; return -1; }
  if (init_qpos) for (size_t i = 0; i < (size_t)n * nq; i++) if (!std::isfinite(init_qpos[i])) { s->err = "fb_ik_solve: non-finite init_qpos"; return -1; }
  dev_select(s);
  if (sync_stream(s) != 0) return -2;
  const int Np = s->d.Np;
  std::vector<int> done(Np, 1); std::fill(done.begin(), done.begin() + n, 0);
  std::vector<float> nan(Np, std::numeric_limits<float>::quiet_NaN()), zero((size_t)Np * p.n_fdof, 0.0f);
  std::vector<int> zi(Np, 0);
  copy_async(s, (void*)p.target, target_xpos, sizeof(float) * (size_t)n * nt);
  copy_async(s, p.u, zero.data(), sizeof(float) * zero.size()); copy_async(s, p.step, zi.data(), sizeof(int) * Np);
  copy_async(s, p.done, done.data(), sizeof(int) * Np); copy_async(s, p.err, nan.data(), sizeof(float) * Np);
  copy_async(s, p.err_first, nan.data(), sizeof(float) * Np); copy_async(s, p.steps, zi.data(), sizeof(int) * Np);
  std::vector<unsigned char> zb(Np, 0); copy_async(s, p.success, zb.data(), Np);
  if (init_qpos && copy_rows_async(s, s->d.qpos, (size_t)s->d.rec * 4, init_qpos, (size_t)nq * 4, (size_t)nq * 4, n) != 0) return -2;
  if (sync_stream(s) != 0) return -2;           // the host vectors go out of scope below
  p.n = n; s->ik_solved = n;
  for (int live = n; live > 0;) if (ik_launch(s, &live) != 0) return -2;
  return 0;
}

int fb_ik_read(FbHandle s, float* qpos, float* err, float* err_first, int32_t* steps, uint8_t* success) {
  if (!s) return -1;
  const DevIk& p = s->ik;
  if (!p.live || s->ik_solved < 1) { s->err = "fb_ik_read: no IK solve to read"; return -1; }
  if (sync_stream(s) != 0) return -2;
  const size_t n = s->ik_solved, nq = s->m.nq;
  return read_out(s, {{qpos, s->d.qpos, (size_t)s->d.rec * 4, nq * 4, n}, {err, p.err, 0, 4 * n, 1}, {err_first, p.err_first, 0, 4 * n, 1},
                      {steps, p.steps, 0, 4 * n, 1}, {success, p.success, 0, n, 1}});
}

}  // extern "C"

// -------------------------------------------------------------------------------------------
// inverse dynamics (fb_inverse*; fb_inverse.h): its own kernel parameter (DevInv) and buffers (inv_scope), allocated on first use
struct InvWarp {
  DevModel m; DevData d; DevInv p;
  FB_DEVM void operator()(unsigned char* sh, int e) const { kinv_run(m, d, p, reinterpret_cast<float*>(sh), e); }
};
static void launch_inv(FbSim* s, const DevInv& p) { warp_launch(s, "inverse", p.n, sizeof(float) * FB_INV_SH, InvWarp{s->m, s->d, p}); }
static int inv_alloc(FbSim* s) {
  if (s->inv.qacc) return 0;
  const size_t Np = (size_t)s->d.Np, nv = (size_t)s->m.nv;
  DevInv& p = s->inv;
  if (int rc = scope_alloc(s, s->inv_scope, "out of device memory (inverse dynamics)", [&] {
        p.qacc = dalloc<float>(s, Np * nv); p.qfrc_inverse = dalloc<float>(s, Np * nv); p.qfrc_constraint = dalloc<float>(s, Np * nv);
        p.efc_force = dalloc<float>(s, Np * FB_MAXEFC); })) {
    s->inv = DevInv{}; return rc; }
  return 0;
}
// the sensor pass of an inverse (fb_inverse.h kinv_sensors) over its p.n envs; a model without sensordata launches nothing
struct InvSensWarp {
  DevModel m; DevData d; DevInvSens p;
  FB_DEVM void operator()(unsigned char* sh, int e) const { kinv_sensors(m, d, p, reinterpret_cast<float*>(sh), e); }
};
static size_t inv_sens_slice(const FbSim* s) { return slice_bytes(0, FB_INVS_SH(s->m.nbody)); }
static void launch_inv_sensors(FbSim* s, const DevInv& inv, float* sensordata) {
  if (s->m.nsensordata > 0) warp_launch(s, "inverse_sensors", inv.n, inv_sens_slice(s), InvSensWarp{s->m, s->d, DevInvSens{inv, sensordata}});
}

extern "C" {

int fb_query_sensors(FbHandle s, int on) {
  if (!s) return -1;
  if (on && inv_sens_slice(s) * FB_WPB > 48 * 1024) {
    s->err = "fb_query_sensors: the sensor pass keeps 18 floats per body in shared memory, and " + std::to_string(s->m.nbody) + " bodies do not fit";
    return -1;
  }
  s->sens_on = on != 0;
  return 0;
}

int fb_inverse(FbHandle s, int n, const float* qacc, int is_device) {
  if (!s) return -1;
  if (n < 1 || n > s->d.N) { s->err = "fb_inverse: 1 <= n <= n_envs problems"; return -1; }
  if (!qacc) { s->err = "fb_inverse: qacc is NULL"; return -1; }
  const size_t cnt = (size_t)n * s->m.nv;
  if (!is_device) for (size_t i = 0; i < cnt; i++) if (!std::isfinite(qacc[i])) { s->err = "fb_inverse: non-finite qacc"; return -1; }
  dev_select(s);
  if (int rc = inv_alloc(s)) return rc;
  const bool sens = s->sens_on != 0;
  if (sens && !s->inv_sd) {
    if (int rc = scope_alloc(s, s->inv_sd_scope, "out of device memory (inverse sensordata)",
                             [&] { s->inv_sd = dalloc<float>(s, (size_t)s->d.Np * s->m.nsensordata); })) { s->inv_sd = nullptr; return rc; }
  }
  DevInv& p = s->inv;
  if (copy_async(s, p.qacc, qacc, sizeof(float) * cnt) != 0) return -2;
  p.n = n;
  launch_step1(s);                             // the position / velocity stage fb_forward runs (sens_mode -1: no sensor sums)
  launch_inv(s, s->inv);
  if (sens) launch_inv_sensors(s, s->inv, s->inv_sd);
  if (launch_check(s, "fb_inverse") != 0) return -2;
  s->inv_done = n; s->inv_sens = sens;
  return is_device ? 0 : sync_stream(s);       // a host qacc may be reused once the call returns
}

int fb_inverse_sensor_read(FbHandle s, float* sensordata, int is_device) {
  if (!s) return -1;
  if (s->inv_done < 1) { s->err = "fb_inverse_sensor_read: no inverse to read (fb_inverse)"; return -1; }
  if (!s->inv_sens) { s->err = "fb_inverse_sensor_read: the last fb_inverse ran with sensors off (fb_query_sensors)"; return -1; }
  return read_out(s, {{sensordata, s->inv_sd, 0, 4 * (size_t)s->inv_done * s->m.nsensordata, 1}});
}

int fb_inverse_read(FbHandle s, float* qfrc_inverse, float* qfrc_constraint, float* efc_force, int is_device) {
  if (!s) return -1;
  const DevInv& p = s->inv;
  if (s->inv_done < 1) { s->err = "fb_inverse_read: no inverse to read (fb_inverse)"; return -1; }
  const size_t n = (size_t)s->inv_done, nv = (size_t)s->m.nv;
  return read_out(s, {{qfrc_inverse, p.qfrc_inverse, 0, 4 * n * nv, 1}, {qfrc_constraint, p.qfrc_constraint, 0, 4 * n * nv, 1},
                      {efc_force, p.efc_force, 0, 4 * n * FB_MAXEFC, 1}});
}

}  // extern "C"

// -------------------------------------------------------------------------------------------
// finite-difference Jacobians (fb_fd_*; fb_fd.h): the four queries run one path.  Each keeps its own outputs, so a query's results can
// be read after another has run; the scratch (FdScratch) is shared
struct FdPerturb {
  DevModel m; DevData d; DevFdQ p;
  FB_DEVM void operator()(unsigned char*, int e) const { kfd_perturb(m, d, p, e); }
};
struct FdDiff {
  DevModel m; DevData d; DevFdQ p;
  FB_DEVM void operator()(unsigned char*, int w) const { kfd_diff(m, d, p, w); }
};
struct FdRows {
  DevData d; DevFdQ p;
  FB_DEVM void operator()(unsigned char*, int w) const { kfd_rows(d, p, w); }
};
template <bool ACC> struct FdSnap {
  DevModel m; DevData d; float* snap;
  FB_DEVM void operator()(unsigned char*, int e) const { kfd_snap(m, d, snap, e, ACC); }
};
template <typename F> static bool all_finite(const F* x, size_t n) { for (size_t i = 0; i < n; i++) if (!std::isfinite(x[i])) return false; return true; }
// the inputs of one problem: (dq, qvel, act, ctrl), (dq, qvel, qacc) or the program's directions; and the envs it takes
static int fd_inputs(const FbSim* s, const FdQuery& q) { return q.param ? s->fdp_k : q.inverse ? 3 * s->m.nv : 2 * s->m.nv + s->m.na + s->m.nu; }
static int fd_columns(const FbSim* s, const FdQuery& q, int centered) { return 1 + (centered ? 2 : 1) * fd_inputs(s, q); }
// the problems of a transition query: written bank rows, none saved while its env was held for a reset
static int fd_slots_valid(FbSim* s, const char* who, const int32_t* slots, int n) {
  for (int k = 0; k < n; k++) {
    const int sl = slots[k];
    if (sl < 0 || sl >= s->st_slots) { s->err = std::string(who) + ": slot out of range of the bank"; return -1; }
    if (!s->st_written[sl]) { s->err = std::string(who) + ": slot " + std::to_string(sl) + " was never written"; return -1; }
    if (s->st_written[sl] == 2) { s->err = std::string(who) + ": slot " + std::to_string(sl) + " was saved while its env was held for a reset (a held env does not integrate)"; return -1; }
  }
  return 0;
}
// the slot of every env (its problem's; the envs past the problems take the last problem's), uploaded as a device list
static int fan_out_ids(FbSim* s, const int32_t* slots, int n, int ncol, const int** slot_dev) {
  const int N = s->d.N;
  std::vector<int32_t> fan(N);
  for (int e = 0; e < N; e++) fan[e] = slots[std::min(e / ncol, n - 1)];
  const int* ed;
  return state_ids(s, nullptr, fan.data(), N, &ed, slot_dev);
}
// every env a copy of its problem's row, warm start included; the envs past the problems copy the last problem's
static int fd_fan_out(FbSim* s, const int32_t* slots, int n, int ncol) {
  const int* sd;
  if (int rc = fan_out_ids(s, slots, n, ncol, &sd)) return rc;
  launch_state<true>(s, nullptr, sd, s->d.N);
  return 0;
}

// the arguments of a compute entry: n problems (bank slots of a transition; host or device rows qpos, qvel, qacc of an inverse)
struct FdCall { int n; const int32_t* slots; const float* in[3]; float eps; int centered, n_substeps, is_device; };
static int fd_check(FbSim* s, const FdQuery& q, const FdCall& c) {
  const std::string who = q.name;
  if (q.inverse && !q.param && s->d.prm) {
    s->err = who + ": the handle has a parameter overlay, and the columns are written from qpos, qvel and qacc alone (fb_param_clear first)"; return -1; }
  if (q.param && !s->d.prm) {
    s->err = who + ": the handle has no parameter overlay, and the columns nudge each problem's own parameters: " +
             (q.inverse ? "fb_param_set first (problem i takes env i's parameters)" : "fb_param_set first, then fb_state_bank and fb_state_save the rows");
    return -1; }
  if (q.param && s->fdp_k < 1) { s->err = who + ": no direction program (fb_fd_param_program)"; return -1; }
  if (!q.inverse && state_ready(s, q.name) != 0) return -1;
  const int N = s->d.N, ncol = fd_columns(s, q, c.centered);
  if ((!q.inverse && !c.slots) || c.n < 1 || (long long)c.n * ncol > N) {
    s->err = who + ": 1 <= n problems with n * " + q.cols + " (" + std::to_string(ncol) + ") <= n_envs (" + std::to_string(N) + ")"; return -1; }
  if (q.inverse) {
    if (!c.in[0] || !c.in[1] || !c.in[2]) { s->err = who + ": qpos, qvel and qacc must not be NULL"; return -1; }
    const size_t cnt[3] = {(size_t)c.n * s->m.nq, (size_t)c.n * s->m.nv, (size_t)c.n * s->m.nv};
    const char* what[3] = {"qpos", "qvel", "qacc"};
    if (!c.is_device) for (int t = 0; t < 3; t++) if (!all_finite(c.in[t], cnt[t])) { s->err = who + ": non-finite " + what[t]; return -1; }
  }
  if (!(c.eps > 0.0f) || !std::isfinite(c.eps)) { s->err = who + ": eps must be positive and finite"; return -1; }
  if (q.param && s->fdp_scale && !(c.eps < 1.0f)) { s->err = who + ": the program has scale directions, which need eps < 1"; return -1; }
  if (!q.inverse && c.n_substeps < 1) { s->err = who + ": n_substeps >= 1"; return -1; }
  return q.inverse ? 0 : fd_slots_valid(s, q.name, c.slots, c.n);
}
// the parts of the shared scratch a call of q needs, allocated on first use
static int fd_scratch(FbSim* s, const FdQuery& q, bool sens) {
  FdScratch x = s->fdx;                        // kept once every part this call adds is there
  const size_t Np = s->d.Np, half = std::max(1, s->d.N / 2), nq = s->m.nq, nv = s->m.nv;
  std::vector<void*> scope;
  if (int rc = scope_alloc(s, scope, "out of device memory (finite-difference scratch)", [&] {
        if (!x.delta) x.delta = dalloc<float>(s, Np);
        if (q.inverse && !x.inv.qacc) {
          x.inv.qacc = dalloc<float>(s, Np * nv); x.inv.qfrc_inverse = dalloc<float>(s, Np * nv);
          x.inv.qfrc_constraint = dalloc<float>(s, Np * nv); x.inv.efc_force = dalloc<float>(s, Np * FB_MAXEFC);
          x.qpos = dalloc<float>(s, half * nq); x.qvel = dalloc<float>(s, half * nv); x.qacc = dalloc<float>(s, half * nv);
        }
        if (q.inverse && q.param && !x.rows) x.rows = dalloc<float>(s, half * s->d.prm_stride);
        if (sens && !x.sens) x.sens = dalloc<float>(s, Np * s->m.nsensordata); }))
    return rc;
  s->fdx = x;
  return 0;
}
// the outputs of a call of nin inputs, their pointers aside: a block per range of inputs ((dq, qvel, act) and ctrl; dq, qvel and qacc;
// the directions) and per source (the state or qfrc_inverse, qM for the dq inputs of the state inverse, the sensors), then the nominal
// column's.  The sensor blocks are empty when sens is off.
static void fd_layout(FbSim* s, FdQuery& q, int nin, bool sens) {
  const DevModel& m = s->m;
  const int nv = m.nv, nx = 2 * nv + m.na, nsd = sens ? m.nsensordata : 0;
  const int nparts = q.param ? 1 : q.inverse ? 3 : 2, part[3] = {q.param ? nin : q.inverse ? nv : nx, q.inverse ? nv : m.nu, nv};
  const float *src = q.inverse ? s->fdx.inv.qfrc_inverse : nullptr, *sd = s->fdx.sens;
  DevFdQ& p = q.p;
  p.nblk = 0;
  auto blk = [&](const float* f, int stride, int L, int j0, int w, bool sensor) {
    FdBlock& k = p.blk[p.nblk++];
    k = FdBlock{f, (unsigned)stride, L, j0, w, q.inverse, sensor, k.out};
  };
  for (int t = 0, j0 = 0; t < nparts; j0 += part[t++]) blk(src, nv, q.inverse ? nv : nx, j0, part[t], false);
  if (q.inverse && !q.param) blk(s->d.qM, s->d.rec, m.nM, 0, nv, false);
  for (int t = 0, j0 = 0; t < nparts; j0 += part[t++]) blk(sd, nsd, nsd, j0, part[t], true);
  p.nom[0] = FdNom{src, (unsigned)nv, q.inverse ? nv : m.nq + nv + m.na, p.nom[0].out};
  p.nom[1] = FdNom{sd, (unsigned)nsd, nsd, p.nom[1].out};
}
// the outputs (sens: the sensor outputs), allocated once for every call the capacity rule admits: a problem takes 1 + nin envs or more,
// so n nin < N and n <= N / 2.  A program's k is not known beforehand: its blocks (w = k) take the bound N - 1 of n k.
static int fd_outputs(FbSim* s, FdQuery& q, int nin, bool sens) {
  std::vector<void*>& scope = sens ? q.sens_scope : q.scope;
  if (!scope.empty()) return 0;
  const int N = s->d.N;
  const size_t cap = std::max(1, q.param ? N / 2 : std::min(N / 2, (N - 1) / nin)), all = std::max(1, N - 1);
  DevFdQ p = q.p;
  if (int rc = scope_alloc(s, scope, sens ? "out of device memory (finite-difference sensor outputs)" : "out of device memory (finite-difference outputs)", [&] {
        for (int o = 0; o < p.nblk; o++)
          if (p.blk[o].sensor == sens) p.blk[o].out = dalloc<float>(s, p.blk[o].L * (q.param ? all : cap * p.blk[o].w));
        p.nom[sens].out = dalloc<float>(s, cap * p.nom[sens].L); }))
    return rc;
  q.p = p;
  return 0;
}
// a compute entry: the checks, scratch and outputs, the problems into the envs (the fan-out of bank rows, or an inverse's rows), then
// perturb, evaluate and difference
static int fd_run(FbSim* s, FdQuery& q, const FdCall& c) {
  if (fd_check(s, q, c) != 0) return -1;
  const int N = s->d.N, n = c.n, nin = fd_inputs(s, q), ncol = fd_columns(s, q, c.centered);
  const bool sens = s->sens_on != 0, snap = sens && s->m.nsensordata > 0;
  q.done = 0;
  dev_select(s);
  if (int rc = fd_scratch(s, q, sens)) return rc;
  fd_layout(s, q, nin, sens);
  if (int rc = fd_outputs(s, q, nin, false)) return rc;
  if (sens) if (int rc = fd_outputs(s, q, nin, true)) return rc;
  const FdScratch& x = s->fdx;
  if (!q.inverse) { if (int rc = fd_fan_out(s, c.slots, n, ncol)) return rc; }
  else if (copy_async(s, x.qpos, c.in[0], sizeof(float) * n * s->m.nq) != 0 || copy_async(s, x.qvel, c.in[1], sizeof(float) * n * s->m.nv) != 0 ||
           copy_async(s, x.qacc, c.in[2], sizeof(float) * n * s->m.nv) != 0) return -2;
  DevFdQ& p = q.p;
  p.n = n; p.ncol = ncol; p.nin = nin; p.centered = c.centered != 0; p.eps = c.eps; p.delta = x.delta;
  p.ju = q.inverse || q.param ? nin : 2 * s->m.nv + s->m.na;
  p.g = q.param ? s->fdp_prog : DevFdPrmProg{};
  p.qpos = q.inverse ? x.qpos : nullptr; p.qvel = x.qvel; p.qacc = x.qacc;
  p.rows = q.inverse && q.param ? x.rows : nullptr;
  p.inv = x.inv; p.inv.n = n * ncol;
  if (p.rows) warp_launch(s, "fd_rows", n, 0, FdRows{s->d, p});
  warp_launch(s, "fd_perturb", N, 0, FdPerturb{s->m, s->d, p});
  launch_step1(s);                             // the position / velocity stage of the nudged states (an inverse's as fb_inverse runs it)
  if (q.inverse) {
    launch_inv(s, p.inv);
    if (sens) launch_inv_sensors(s, p.inv, x.sens);
  } else if (!snap) {
    step_run(s, c.n_substeps);                 // fb_step's launches
  } else {                                     // the same, split after the first substep to snapshot the sensors of x
    warp_launch(s, "fd_snap", n * ncol, 0, FdSnap<false>{s->m, s->d, x.sens});
    step_run(s, 1);
    warp_launch(s, "fd_snap", n * ncol, 0, FdSnap<true>{s->m, s->d, x.sens});
    if (c.n_substeps > 1) step_run(s, c.n_substeps - 1);
  }
  warp_launch(s, "fd_diff", n * nin, 0, FdDiff{s->m, s->d, p});
  if (launch_check(s, q.name) != 0) return -2;
  q.done = n; q.sens = sens; q.at = s->launches;
  return q.inverse && c.is_device ? 0 : sync_stream(s);   // host rows may be reused once the call returns; the fan-out list is a host vector
}
// a read entry: the outputs (sens: the sensor outputs) in the entry's order, the blocks and then the nominal column's (the next state:
// qpos, qvel, act)
static int fd_read(FbSim* s, const FdQuery& q, const char* who, bool sens, std::initializer_list<void*> dst) {
  if (q.done < 1) { s->err = std::string(who) + ": no " + q.what + " to read (" + q.name + ")"; return -1; }
  if (sens && !q.sens) { s->err = std::string(who) + ": the last " + q.name + " ran with sensors off (fb_query_sensors)"; return -1; }
  const size_t n = q.done;
  const DevFdQ& p = q.p;
  void* const* d = dst.begin();
  std::vector<ReadOut> outs;
  for (int o = 0; o < p.nblk; o++) if (p.blk[o].sensor == sens) outs.push_back({*d++, p.blk[o].out, 0, 4 * n * p.blk[o].L * p.blk[o].w, 1});
  const FdNom& c = p.nom[sens];
  if (c.src || sens) outs.push_back({*d, c.out, 0, 4 * n * c.L, 1});
  else {
    const size_t w[3] = {(size_t)s->m.nq, (size_t)s->m.nv, (size_t)s->m.na};
    for (size_t t = 0, at = 0; t < 3; at += w[t++]) outs.push_back({d[t], c.out + at, 4 * (size_t)c.L, 4 * w[t], n});
  }
  return read_out(s, outs);
}

extern "C" {

int fb_fd_columns(FbHandle s, int centered) { return s ? fd_columns(s, s->fd_tr, centered) : -1; }
int fb_fd_inverse_columns(FbHandle s, int centered) { return s ? fd_columns(s, s->fd_inv, centered) : -1; }

int fb_fd_transition(FbHandle s, const int32_t* slots, int n, float eps, int centered, int n_substeps) {
  return s ? fd_run(s, s->fd_tr, {n, slots, {}, eps, centered, n_substeps, 0}) : -1;
}
int fb_fd_read(FbHandle s, float* A, float* B, float* qpos_next, float* qvel_next, float* act_next, int is_device) {
  return s ? fd_read(s, s->fd_tr, "fb_fd_read", false, {A, B, qpos_next, qvel_next, act_next}) : -1;
}
int fb_fd_sensor_read(FbHandle s, float* C, float* D, float* sensordata, int is_device) {
  return s ? fd_read(s, s->fd_tr, "fb_fd_sensor_read", true, {C, D, sensordata}) : -1;
}

int fb_fd_inverse(FbHandle s, int n, const float* qpos, const float* qvel, const float* qacc, float eps, int centered, int is_device) {
  return s ? fd_run(s, s->fd_inv, {n, nullptr, {qpos, qvel, qacc}, eps, centered, 1, is_device}) : -1;
}
int fb_fd_inverse_read(FbHandle s, float* DfDq, float* DfDv, float* DfDa, float* DmDq, float* qfrc_inverse, int is_device) {
  return s ? fd_read(s, s->fd_inv, "fb_fd_inverse_read", false, {DfDq, DfDv, DfDa, DmDq, qfrc_inverse}) : -1;
}
int fb_fd_inverse_sensor_read(FbHandle s, float* DsDq, float* DsDv, float* DsDa, float* sensordata, int is_device) {
  return s ? fd_read(s, s->fd_inv, "fb_fd_inverse_sensor_read", true, {DsDq, DsDv, DsDa, sensordata}) : -1;
}

int fb_fd_param_program(FbHandle s, int k, const int32_t* kind, const int32_t* dir_ptr, const int32_t* param, const int32_t* elem, const float* floor) {
  if (!s) return -1;
  const char* who = "fb_fd_param_program: ";
  if (k < 0) { s->err = std::string(who) + "k >= 1 directions (0 clears the program)"; return -1; }
  if (k > 0 && (!kind || !dir_ptr || !param || !elem || !floor)) { s->err = std::string(who) + "kind, dir_ptr, param, elem and floor must not be NULL"; return -1; }
  if (k > 0 && dir_ptr[0] != 0) { s->err = std::string(who) + "dir_ptr[0] must be 0"; return -1; }
  std::vector<int> kd(k), ptr(k + 1, 0), slot, mslot, nonneg; std::vector<float> fl;
  bool scale = false;
  for (int j = 0; j < k; j++) {
    const int a = dir_ptr[j], b = dir_ptr[j + 1], dj = kind[j];
    const std::string at = "direction " + std::to_string(j) + ": ";
    if (dj != FB_FD_ELEMENT && dj != FB_FD_SCALE) { s->err = who + at + "kind is 0 (element) or 1 (scale)"; return -1; }
    if (b <= a) { s->err = who + at + "no entries (dir_ptr must increase)"; return -1; }
    if (dj == FB_FD_ELEMENT && b != a + 1) { s->err = who + at + "an element direction has one entry"; return -1; }
    scale = scale || dj == FB_FD_SCALE;
    std::vector<int> seen;
    for (int t = a; t < b; t++) {
      const int p = param[t], i = elem[t];
      if (p < 0 || p >= FB_NPARAMS) { s->err = who + at + "unknown parameter " + std::to_string(p); return -1; }
      if (i < 0 || i >= s->prm_n[p]) { s->err = who + at + "element " + std::to_string(i) + " out of range of parameter " + std::to_string(p) + " (fb_param_size " + std::to_string(s->prm_n[p]) + ")"; return -1; }
      if (p == FB_P_JNT_STIFFNESS && s->h_jnt_type[i] != FB_JNT_HINGE) {
        s->err = who + at + "joint " + std::to_string(i) + " is not a hinge: the step has springs on hinge joints only"; return -1; }
      if (dj == FB_FD_ELEMENT && !(std::isfinite(floor[t]) && floor[t] > 0.0f)) { s->err = who + at + "the floor must be positive and finite"; return -1; }
      const int sl = s->d.prm_off[p] + prm_slot(p, i);
      if (std::find(seen.begin(), seen.end(), sl) != seen.end()) { s->err = who + at + "an element appears twice"; return -1; }
      seen.push_back(sl);
      slot.push_back(sl);
      mslot.push_back(p == FB_P_DOF_DAMPING ? s->d.prm_mdamp + s->h_dof_Madr[i] : -1);
      nonneg.push_back(p != FB_P_ACTUATOR_GAINPRM && p != FB_P_ACTUATOR_BIASPRM && p != FB_P_GRAVITY && p != FB_P_WIND);
      fl.push_back(dj == FB_FD_ELEMENT ? floor[t] : 1.0f);
    }
    kd[j] = dj; ptr[j + 1] = b;
  }
  if (sync_stream(s) != 0) return -2;          // a call in flight may still read the old tables
  scope_free(s, s->fdp_prog_scope);
  s->fdp_prog = DevFdPrmProg{}; s->fdp_k = 0; s->fdp_scale = false;
  if (k == 0) return 0;
  DevFdPrmProg& g = s->fdp_prog;
  if (int rc = scope_alloc(s, s->fdp_prog_scope, "out of device memory (parameter direction program)", [&] {
        g.kind = up(s, kd); g.ptr = up(s, ptr); g.slot = up(s, slot); g.mslot = up(s, mslot); g.nonneg = up(s, nonneg); g.floor = up(s, fl); })) {
    g = DevFdPrmProg{}; return rc; }
  s->fdp_k = k; s->fdp_scale = scale;
  return 0;
}

int fb_fd_param_columns(FbHandle s, int centered) {
  if (!s) return -1;
  if (s->fdp_k < 1) { s->err = "fb_fd_param_columns: no direction program (fb_fd_param_program)"; return -1; }
  return fd_columns(s, s->fd_ptr, centered);
}

int fb_fd_param_transition(FbHandle s, const int32_t* slots, int n, float eps, int centered, int n_substeps) {
  return s ? fd_run(s, s->fd_ptr, {n, slots, {}, eps, centered, n_substeps, 0}) : -1;
}
int fb_fd_param_read(FbHandle s, float* dxdp, float* qpos_next, float* qvel_next, float* act_next, int is_device) {
  return s ? fd_read(s, s->fd_ptr, "fb_fd_param_read", false, {dxdp, qpos_next, qvel_next, act_next}) : -1;
}
int fb_fd_param_sensor_read(FbHandle s, float* dsdp, float* sensordata, int is_device) {
  return s ? fd_read(s, s->fd_ptr, "fb_fd_param_sensor_read", true, {dsdp, sensordata}) : -1;
}

int fb_fd_param_inverse(FbHandle s, int n, const float* qpos, const float* qvel, const float* qacc, float eps, int centered, int is_device) {
  return s ? fd_run(s, s->fd_pinv, {n, nullptr, {qpos, qvel, qacc}, eps, centered, 1, is_device}) : -1;
}
int fb_fd_param_inverse_read(FbHandle s, float* DfDp, float* qfrc_inverse, int is_device) {
  return s ? fd_read(s, s->fd_pinv, "fb_fd_param_inverse_read", false, {DfDp, qfrc_inverse}) : -1;
}
int fb_fd_param_inverse_sensor_read(FbHandle s, float* DsDp, float* sensordata, int is_device) {
  return s ? fd_read(s, s->fd_pinv, "fb_fd_param_inverse_sensor_read", true, {DsDp, sensordata}) : -1;
}

}  // extern "C"

// -------------------------------------------------------------------------------------------
// rollouts (fb_rollout*; fb_rollout.h): their own kernel parameter (DevRoll) and buffers, allocated on first use and grown with n T
struct RollInput {
  DevModel m; DevData d; DevRoll p; const int* law;
  FB_DEVM void operator()(unsigned char* sh, int e) const { kroll_input(m, d, p, law, reinterpret_cast<float*>(sh), e); }
};
struct RollRecord {
  DevModel m; DevData d; DevRoll p;
  FB_DEVM void operator()(unsigned char*, int e) const { kroll_record(m, d, p, e); }
};
// the feedback bank (fb_rollout_feedback_bank; fb_rollout_feedback is L = 1 without a law list)
static int rollout_feedback(FbSim* s, const char* who, int L, int T, const float* xref, const float* K, const int32_t* law, int n, int is_device) {
  const DevModel& m = s->m;
  const std::string w = who;
  const size_t nx = 2 * (size_t)m.nv + m.na, nr = (size_t)m.nq + m.nv + m.na;
  const bool clear = T == 0 || (!xref && !K);
  if (!clear && (T < 1 || !xref || !K)) { s->err = w + ": T >= 1 steps with both xref and K (T = 0, or both NULL, clears the law)"; return -1; }
  if (!clear && L < 1) { s->err = w + ": L >= 1 laws"; return -1; }
  if (!clear && law && n < 1) { s->err = w + ": a law list of n >= 1 rollouts"; return -1; }
  if (!clear && !law && L != 1) { s->err = w + ": a bank of " + std::to_string(L) + " laws needs a law list"; return -1; }
  if (!clear && law)
    for (int i = 0; i < n; i++)
      if (law[i] < 0 || law[i] >= L) { s->err = w + ": law[" + std::to_string(i) + "] = " + std::to_string(law[i]) + " is outside [0, L = " + std::to_string(L) + ")"; return -1; }
  if (!clear && slice_bytes(0, nx) * FB_WPB > 48 * 1024) {
    s->err = w + ": the input kernel keeps the tangent (2 nv + na = " + std::to_string(nx) + " floats) in shared memory, and it does not fit"; return -1; }
  const size_t lt = (size_t)L * T;
  if (!clear && !is_device && (!all_finite(xref, lt * nr) || !all_finite(K, lt * m.nu * nx))) { s->err = w + ": non-finite xref or K"; return -1; }
  dev_select(s);
  if (sync_stream(s) != 0) return -2;          // a rollout in flight may still read the old law
  s->roll_fb_T = s->roll_fb_L = s->roll_fb_n = 0;
  if (clear) return 0;
  if (int rc = grow(s, who, s->roll_fb_pool, lt, 4 * (nr + m.nu * nx), "feedback laws", "L T", [&](size_t r) {
        s->roll_xref = dalloc<float>(s, r * nr); s->roll_K = dalloc<float>(s, r * m.nu * nx); }))
    return rc;
  if (law) if (int rc = grow(s, who, s->roll_law_pool, n, 4, "law list", "n", [&](size_t r) { s->roll_law = dalloc<int>(s, r); }))
    return rc;
  if (copy_async(s, s->roll_xref, xref, sizeof(float) * lt * nr) != 0 || copy_async(s, s->roll_K, K, sizeof(float) * lt * m.nu * nx) != 0 ||
      (law && copy_async(s, s->roll_law, law, sizeof(int) * n) != 0)) return -2;
  s->roll_fb_T = T; s->roll_fb_L = L; s->roll_fb_n = law ? n : 0;
  return is_device && !law ? 0 : sync_stream(s);   // host arrays may be reused once the call returns
}

extern "C" {

int fb_rollout_feedback(FbHandle s, int T, const float* xref, const float* K, int is_device) {
  return s ? rollout_feedback(s, "fb_rollout_feedback", 1, T, xref, K, nullptr, 0, is_device) : -1;
}

int fb_rollout_feedback_bank(FbHandle s, int L, int T, const float* xref, const float* K, const int32_t* law, int n, int is_device) {
  return s ? rollout_feedback(s, "fb_rollout_feedback_bank", L, T, xref, K, law, n, is_device) : -1;
}

int fb_rollout(FbHandle s, const int32_t* slots, int n, int T, int n_substeps, const float* ctrl, const float* qfrc_applied,
               const float* xfrc_applied, int is_device) {
  if (!s) return -1;
  const char* who = "fb_rollout";
  if (state_ready(s, who) != 0) return -1;
  const int N = s->d.N;
  if (!slots || n < 1 || n > N) { s->err = "fb_rollout: 1 <= n <= n_envs (" + std::to_string(N) + ") rollouts, each with its slot"; return -1; }
  if (T < 1) { s->err = "fb_rollout: T >= 1 control steps"; return -1; }
  if (n_substeps < 1) { s->err = "fb_rollout: n_substeps >= 1"; return -1; }
  if (!ctrl) { s->err = "fb_rollout: ctrl is NULL"; return -1; }
  const bool app = qfrc_applied || xfrc_applied;
  if (app && !s->d.qfrc_applied) {
    s->err = "fb_rollout: applied-force sequences need the handle's applied-force arrays, which the state rows carry: allocate them (fb_applied_ptrs) before fb_state_bank";
    return -1; }
  if (s->roll_fb_T && s->roll_fb_T != T) {
    s->err = "fb_rollout: the feedback law has " + std::to_string(s->roll_fb_T) + " steps and the call " + std::to_string(T) + " (fb_rollout_feedback)"; return -1; }
  if (s->roll_fb_n && s->roll_fb_n != n) {
    s->err = "fb_rollout: the law list has " + std::to_string(s->roll_fb_n) + " rollouts and the call " + std::to_string(n) + " (fb_rollout_feedback_bank)"; return -1; }
  if (fd_slots_valid(s, who, slots, n) != 0) return -1;
  const DevModel& m = s->m;
  const size_t rows = (size_t)n * T, nq = m.nq, nv = m.nv, na = m.na, nu = m.nu, nsd = m.nsensordata, nxf = 6 * (size_t)m.nbody;
  if (!is_device) {
    if (!all_finite(ctrl, rows * nu)) { s->err = "fb_rollout: non-finite ctrl"; return -1; }
    if ((qfrc_applied && !all_finite(qfrc_applied, rows * nv)) || (xfrc_applied && !all_finite(xfrc_applied, rows * nxf))) {
      s->err = "fb_rollout: non-finite applied force"; return -1; }
  }
  dev_select(s);
  s->roll_done = 0;
  DevRoll& p = s->roll;
  if (int rc = grow(s, who, s->roll_pool, rows, 4 * (2 * nu + nq + nv + na + 2), "records", "n T", [&](size_t r) {
        p.ctrl = dalloc<float>(s, r * nu); p.qpos = dalloc<float>(s, r * nq); p.qvel = dalloc<float>(s, r * nv); p.act = dalloc<float>(s, r * na);
        p.ctrl_out = dalloc<float>(s, r * nu); p.time = dalloc<float>(s, r); p.flags = dalloc<int>(s, r); }))
    return rc;
  if (int rc = app ? grow(s, who, s->roll_app_pool, rows, 4 * (nv + nxf), "applied-force inputs", "n T", [&](size_t r) {
        s->roll_qf = dalloc<float>(s, r * nv); s->roll_xf = dalloc<float>(s, r * nxf); }) : 0)
    return rc;
  const bool sens = s->sens_on != 0;
  if (int rc = sens ? grow(s, who, s->roll_sd_pool, rows, 8 * nsd, "sensor records", "n T", [&](size_t r) {
        s->roll_sd = dalloc<float>(s, r * nsd); s->roll_sm = dalloc<float>(s, r * nsd); }) : 0)
    return rc;
  p.qfrc = qfrc_applied ? s->roll_qf : nullptr; p.xfrc = xfrc_applied ? s->roll_xf : nullptr;
  p.sensordata = sens ? s->roll_sd : nullptr; p.sensor_mean = sens ? s->roll_sm : nullptr;
  if (copy_async(s, (void*)p.ctrl, ctrl, 4 * rows * nu) != 0 || (qfrc_applied && copy_async(s, (void*)p.qfrc, qfrc_applied, 4 * rows * nv) != 0) ||
      (xfrc_applied && copy_async(s, (void*)p.xfrc, xfrc_applied, 4 * rows * nxf) != 0)) return -2;
  p.n = n; p.T = T; p.nsub = n_substeps;
  p.xref = s->roll_fb_T ? s->roll_xref : nullptr; p.K = s->roll_fb_T ? s->roll_K : nullptr;
  const size_t slice = p.K ? slice_bytes(0, 2 * nv + na) : 0;
  if (int rc = fd_fan_out(s, slots, n, 1)) return rc;
  launch_step1(s);                             // what the rows do not carry, as fb_state_load runs it
  for (int t = 0; t < T; t++) {                // no host synchronisation or copy inside the horizon
    p.t = t;
    warp_launch(s, "rollout_input", N, slice, RollInput{s->m, s->d, p, s->roll_fb_n ? s->roll_law : nullptr});
    step_run(s, n_substeps);                   // fb_step's launches (the step graph)
    warp_launch(s, "rollout_record", n, 0, RollRecord{s->m, s->d, p});
  }
  if (launch_check(s, who) != 0) return -2;
  s->roll_done = n; s->roll_sens = sens;
  return sync_stream(s);                       // (the fan-out list is a host vector)
}

int fb_rollout_read(FbHandle s, float* qpos, float* qvel, float* act, float* ctrl, float* time, int32_t* flags, int is_device) {
  if (!s) return -1;
  if (s->roll_done < 1) { s->err = "fb_rollout_read: no rollout to read (fb_rollout)"; return -1; }
  const DevRoll& p = s->roll;
  const size_t r = (size_t)s->roll_done * p.T;
  return read_out(s, {{qpos, p.qpos, 0, 4 * r * s->m.nq, 1}, {qvel, p.qvel, 0, 4 * r * s->m.nv, 1}, {act, p.act, 0, 4 * r * s->m.na, 1},
                      {ctrl, p.ctrl_out, 0, 4 * r * s->m.nu, 1}, {time, p.time, 0, 4 * r, 1}, {flags, p.flags, 0, 4 * r, 1}});
}

int fb_rollout_sensor_read(FbHandle s, float* sensordata, float* sensor_mean, int is_device) {
  if (!s) return -1;
  if (s->roll_done < 1) { s->err = "fb_rollout_sensor_read: no rollout to read (fb_rollout)"; return -1; }
  if (!s->roll_sens) { s->err = "fb_rollout_sensor_read: the last fb_rollout ran with sensors off (fb_query_sensors)"; return -1; }
  const size_t r = (size_t)s->roll_done * s->roll.T * s->m.nsensordata;
  return read_out(s, {{sensordata, s->roll_sd, 0, 4 * r, 1}, {sensor_mean, s->roll_sm, 0, 4 * r, 1}});
}

}  // extern "C"

// -------------------------------------------------------------------------------------------
// the iLQR backward pass (fb_lqr; fb_lqr.h): its own kernel parameter (DevLqr) and buffers, allocated on first use and grown with L T and L
template <int KIND> struct LqrWarp {
  DevLqr p;
  FB_DEVM void operator()(unsigned char*, int w) const {
    if (KIND == 0) klqr_init(p, w); else if (KIND == 1) klqr_w(p, w); else if (KIND == 2) klqr_h(p, w);
    else if (KIND == 3) klqr_chol(p, w); else if (KIND == 4) klqr_solve(p, w); else klqr_p(p, w);
  }
};
template <int KIND> struct LqrBoxWarp {
  DevLqr p; DevLqrBox b;
  FB_DEVM void operator()(unsigned char*, int w) const { if (KIND == 0) klqr_boxqp(p, b, w); else klqr_solve_box(p, b, w); }
};

// fb_lqr, and fb_lqr_box with bounds (lower and upper non-NULL)
static int lqr_pass(FbSim* s, const char* who, int L, int T, const float* A, const float* B, const double* q, const double* r,
                    const double* Q, const double* R, const double* Qf, const double* mu, const double* lower, const double* upper,
                    int is_device) {
  const DevModel& m = s->m;
  const int nx = 2 * m.nv + m.na, nu = m.nu, nz = nx + nu;
  const std::string w = who;
  const bool box = lower != nullptr;
  if (L < 1 || T < 1) { s->err = w + ": L >= 1 problems of T >= 1 steps"; return -1; }
  if (!A || !B || !q || !r || !Q || !R || !Qf || !mu) { s->err = w + ": A, B, q, r, Q, R, Qf and mu must not be NULL"; return -1; }
  if (nu < 1) { s->err = w + ": the model has no actuators"; return -1; }
  if ((size_t)nz * (nz + 1) >= ((size_t)1 << 31)) {
    s->err = w + ": nx + nu = " + std::to_string(nz) + " is too large for the 32-bit offsets inside a problem's workspace"; return -1; }
  const size_t lt = (size_t)L * T, l1 = (size_t)L * (T + 1);
  if (!is_device) {
    const char* name[8] = {"A", "B", "q", "r", "Q", "R", "Qf", "mu"};
    const bool ok[8] = {all_finite(A, lt * nx * nx), all_finite(B, lt * nx * nu), all_finite(q, l1 * nx), all_finite(r, lt * nu),
                        all_finite(Q, (size_t)nx), all_finite(R, (size_t)nu), all_finite(Qf, (size_t)nx), all_finite(mu, (size_t)L)};
    for (int i = 0; i < 8; i++) if (!ok[i]) { s->err = w + ": non-finite " + name[i]; return -1; }
    for (size_t i = 0; box && i < lt * nu; i++) {
      const char* bad = std::isnan(lower[i]) || std::isnan(upper[i]) ? "a NaN bound" : lower[i] > upper[i] ? "lower > upper"
                        : lower[i] == HUGE_VAL || upper[i] == -HUGE_VAL ? "a bound that excludes every finite du" : nullptr;
      if (bad) {
        s->err = w + ": " + bad + " at [" + std::to_string(i / nu / T) + "][" + std::to_string(i / nu % T) + "][" + std::to_string(i % nu) + "]";
        return -1; }
    }
  }
  dev_select(s);
  s->lqr_done = 0;
  DevLqr& p = s->lqr;
  DevLqrBox& b = s->lqr_b;
  // per problem step (L (T + 1) rows, the last T + 1st unused by A, B, r, K, k): the inputs A, B, q, r and the outputs K, k
  if (int rc = grow(s, who, s->lqr_pool, l1, 4 * ((size_t)nx * nx + (size_t)nx * nu) + 8 * ((size_t)nx + nu + (size_t)nu * nx + nu),
                    "inputs and gains", "L (T + 1)", [&](size_t n) {
        p.A = dalloc<float>(s, n * nx * nx); p.B = dalloc<float>(s, n * nx * nu); p.q = dalloc<double>(s, n * nx); p.r = dalloc<double>(s, n * nu);
        p.K = dalloc<double>(s, n * nu * nx); p.k = dalloc<double>(s, n * nu); }))
    return rc;
  // per problem: the workspace, mu, dV and status (and the shared weights)
  const size_t ws = (size_t)nx * nx + nx + (size_t)nx * (nz + 1) + (size_t)nz * (nz + 1) + (size_t)nu * nu + 2 * (size_t)nu * (nx + 1) + 3;
  if (int rc = grow(s, who, s->lqr_ws_pool, (size_t)L, 8 * ws + 4, "workspace", "L", [&](size_t n) {
        p.P = dalloc<double>(s, n * nx * nx); p.s = dalloc<double>(s, n * nx); p.W = dalloc<double>(s, n * nx * (nz + 1));
        p.H = dalloc<double>(s, n * nz * (nz + 1)); p.C = dalloc<double>(s, n * nu * nu); p.X = dalloc<double>(s, n * nu * (nx + 1));
        p.G = dalloc<double>(s, n * nu * (nx + 1)); p.mu = dalloc<double>(s, n); p.dV = dalloc<double>(s, 2 * n); p.status = dalloc<int>(s, n);
        p.Q = dalloc<double>(s, nx); p.R = dalloc<double>(s, nu); p.Qf = dalloc<double>(s, nx); }))
    return rc;
  if (copy_async(s, (void*)p.A, A, 4 * lt * nx * nx) != 0 || copy_async(s, (void*)p.B, B, 4 * lt * nx * nu) != 0 ||
      copy_async(s, (void*)p.q, q, 8 * l1 * nx) != 0 || copy_async(s, (void*)p.r, r, 8 * lt * nu) != 0 ||
      copy_async(s, (void*)p.Q, Q, 8 * (size_t)nx) != 0 || copy_async(s, (void*)p.R, R, 8 * (size_t)nu) != 0 ||
      copy_async(s, (void*)p.Qf, Qf, 8 * (size_t)nx) != 0 || copy_async(s, (void*)p.mu, mu, 8 * (size_t)L) != 0) return -2;
  if (box) {
    // per problem step: the bounds and the QP's outputs; per problem: the QP's workspace
    if (int rc = grow(s, who, s->lqr_box_pool, lt, 8 * 2 * (size_t)nu + 4 * ((size_t)nu + 2), "bounds and QP records", "L T", [&](size_t n) {
          b.lower = dalloc<double>(s, n * nu); b.upper = dalloc<double>(s, n * nu); b.clamped = dalloc<int>(s, n * nu); b.qp = dalloc<int>(s, 2 * n); }))
      return rc;
    if (int rc = grow(s, who, s->lqr_qp_pool, (size_t)L, 8 * 4 * (size_t)nu + 4 * (size_t)nu, "QP workspace", "L", [&](size_t n) {
          b.x = dalloc<double>(s, n * nu); b.dx = dalloc<double>(s, n * nu); b.g = dalloc<double>(s, n * nu); b.xt = dalloc<double>(s, n * nu);
          b.set = dalloc<int>(s, n * nu); }))
      return rc;
    if (copy_async(s, (void*)b.lower, lower, 8 * lt * nu) != 0 || copy_async(s, (void*)b.upper, upper, 8 * lt * nu) != 0) return -2;
  }
  p.L = L; p.T = T; p.nx = nx; p.nu = nu;
  warp_launch(s, "lqr_init", L, 0, LqrWarp<0>{p});
  for (int t = T - 1; t >= 0; t--) {           // no host synchronisation inside the pass
    p.t = t;
    warp_launch(s, "lqr_w", L * lqr_tiles(nx, nz + 1), 0, LqrWarp<1>{p});
    warp_launch(s, "lqr_h", L * lqr_tiles(nz, nz + 1), 0, LqrWarp<2>{p});
    if (box) {
      warp_launch(s, "lqr_boxqp", L, 0, LqrBoxWarp<0>{p, b});
      warp_launch(s, "lqr_solve_box", L * ((nx + 1 + 31) / 32), 0, LqrBoxWarp<1>{p, b});
    } else {
      warp_launch(s, "lqr_chol", L, 0, LqrWarp<3>{p});
      warp_launch(s, "lqr_solve", L * ((nx + 1 + 31) / 32), 0, LqrWarp<4>{p});
    }
    warp_launch(s, "lqr_p", L * lqr_tiles(nx, nx + 1), 0, LqrWarp<5>{p});
  }
  if (launch_check(s, who) != 0) return -2;
  s->lqr_done = L; s->lqr_box = box;
  return sync_stream(s);                       // host inputs may be reused once the call returns
}

extern "C" {

int fb_lqr(FbHandle s, int L, int T, const float* A, const float* B, const double* q, const double* r, const double* Q, const double* R,
           const double* Qf, const double* mu, int is_device) {
  return s ? lqr_pass(s, "fb_lqr", L, T, A, B, q, r, Q, R, Qf, mu, nullptr, nullptr, is_device) : -1;
}

int fb_lqr_box(FbHandle s, int L, int T, const float* A, const float* B, const double* q, const double* r, const double* Q, const double* R,
               const double* Qf, const double* mu, const double* lower, const double* upper, int is_device) {
  if (!s) return -1;
  if (!lower || !upper) { s->err = "fb_lqr_box: lower and upper must not be NULL"; return -1; }
  return lqr_pass(s, "fb_lqr_box", L, T, A, B, q, r, Q, R, Qf, mu, lower, upper, is_device);
}

int fb_lqr_box_read(FbHandle s, int32_t* clamped, int32_t* qp, int is_device) {
  if (!s) return -1;
  if (s->lqr_done < 1) { s->err = "fb_lqr_box_read: no backward pass to read (fb_lqr_box)"; return -1; }
  if (!s->lqr_box) { s->err = "fb_lqr_box_read: the last backward pass was fb_lqr, without bounds"; return -1; }
  const size_t lt = (size_t)s->lqr.L * s->lqr.T;
  return read_out(s, {{clamped, s->lqr_b.clamped, 0, 4 * lt * s->lqr.nu, 1}, {qp, s->lqr_b.qp, 0, 8 * lt, 1}});
}

int fb_lqr_read(FbHandle s, double* K, double* k, double* dV, int32_t* status, int is_device) {
  if (!s) return -1;
  if (s->lqr_done < 1) { s->err = "fb_lqr_read: no backward pass to read (fb_lqr)"; return -1; }
  const DevLqr& p = s->lqr;
  const size_t lt = (size_t)p.L * p.T;
  return read_out(s, {{K, p.K, 0, 8 * lt * p.nu * p.nx, 1}, {k, p.k, 0, 8 * lt * p.nu, 1}, {dV, p.dV, 0, 16 * (size_t)p.L, 1},
                      {status, p.status, 0, 4 * (size_t)p.L, 1}});
}

}  // extern "C"

// -------------------------------------------------------------------------------------------
// sampling-based MPC (fb_plan; fb_plan.h): its own kernel parameter (DevPlan) and buffers, the samples rolled out through the rollout
// input kernel with a DevRoll of their own
template <int KIND> struct PlanWarp {
  DevModel m; DevData d; DevPlan p;
  FB_DEVM void operator()(unsigned char*, int w) const {
    if (KIND == 0) kplan_sample(m, p, w); else if (KIND == 1) kplan_cost(m, d, p, w); else if (KIND == 2) kplan_weights(p, w);
    else kplan_update(m, p, w);
  }
};

extern "C" {

int fb_plan_program(FbHandle s, const FbPlanProgram* g) {
  if (!s) return -1;
  const DevModel& m = s->m;
  const size_t nx = 2 * (size_t)m.nv + m.na, nu = m.nu;
  const bool clear = !g || g->n_samples == 0;
  if (!clear) {
    if (nu < 1) { s->err = "fb_plan_program: the model has no actuators"; return -1; }
    if (g->n_samples < 2) { s->err = "fb_plan_program: n_samples >= 2 (0 clears the program)"; return -1; }
    if (g->hold < 1) { s->err = "fb_plan_program: hold >= 1 control steps per knot"; return -1; }
    if (!g->sigma || !g->Q || !g->R || !g->Qf) { s->err = "fb_plan_program: sigma, Q, R and Qf must not be NULL"; return -1; }
    if (!(g->temperature >= 0.0) || !std::isfinite(g->temperature)) { s->err = "fb_plan_program: the temperature must be >= 0 and finite"; return -1; }
    const void* arr[4] = {g->sigma, g->Q, g->R, g->Qf};
    const size_t cnt[4] = {nu, nx, nu, nx};
    const char* name[4] = {"sigma", "Q", "R", "Qf"};
    for (int k = 0; k < 4; k++)
      for (size_t i = 0; i < cnt[k]; i++) {
        const double v = k ? ((const double*)arr[k])[i] : (double)((const float*)arr[k])[i];
        if (!(v >= 0.0) || !std::isfinite(v)) { s->err = std::string("fb_plan_program: ") + name[k] + " must be >= 0 and finite"; return -1; }
      }
  }
  dev_select(s);
  if (sync_stream(s) != 0) return -2;          // a plan in flight may still read the old weights
  scope_free(s, s->plan_prog_scope);
  DevPlan& p = s->plan;
  p.K = 0; p.sigma = nullptr; p.Q = p.R = p.Qf = nullptr;
  s->plan_done = 0;
  if (clear) return 0;
  if (int rc = scope_alloc(s, s->plan_prog_scope, "fb_plan_program: out of device memory", [&] {
        p.sigma = up(s, std::vector<float>(g->sigma, g->sigma + nu)); p.Q = up(s, std::vector<double>(g->Q, g->Q + nx));
        p.R = up(s, std::vector<double>(g->R, g->R + nu)); p.Qf = up(s, std::vector<double>(g->Qf, g->Qf + nx)); })) {
    p.sigma = nullptr; p.Q = p.R = p.Qf = nullptr; return rc; }
  p.K = g->n_samples; p.hold = g->hold; p.temperature = g->temperature;
  return 0;
}

int fb_plan(FbHandle s, const int32_t* slots, int L, int T, int n_substeps, int n_iter, const uint32_t* seeds, const float* mean,
            const float* xref, const float* uref, int is_device) {
  if (!s) return -1;
  const char* who = "fb_plan";
  if (state_ready(s, who) != 0) return -1;
  DevPlan& p = s->plan;
  if (p.K < 1) { s->err = "fb_plan: no plan program (fb_plan_program)"; return -1; }
  const int N = s->d.N, K = p.K;
  if (L < 1 || (long long)L * K > N) {
    s->err = "fb_plan: 1 <= L problems with L * n_samples (" + std::to_string(K) + ") <= n_envs (" + std::to_string(N) + ")"; return -1; }
  if (T < 1 || n_substeps < 1 || n_iter < 1) { s->err = "fb_plan: T >= 1 control steps, n_substeps >= 1 and n_iter >= 1"; return -1; }
  if (!slots || !seeds || !mean || !xref) { s->err = "fb_plan: slots, seeds, mean and xref must not be NULL"; return -1; }
  if (fd_slots_valid(s, who, slots, L) != 0) return -1;
  const DevModel& m = s->m;
  const size_t nu = m.nu, nr = (size_t)m.nq + m.nv + m.na, lt = (size_t)L * T, l1 = (size_t)L * (T + 1);
  if (!is_device && (!all_finite(mean, lt * nu) || !all_finite(xref, l1 * nr) || (uref && !all_finite(uref, lt * nu)))) {
    s->err = "fb_plan: non-finite mean, xref or uref"; return -1; }
  dev_select(s);
  s->plan_done = 0;
  const size_t n = (size_t)L * K;
  if (int rc = grow(s, who, s->plan_s_pool, n * T, 4 * nu, "samples", "L n_samples T", [&](size_t r) { p.ctrl = dalloc<float>(s, r * nu); }))
    return rc;
  if (int rc = grow(s, who, s->plan_k_pool, n, 16, "sample costs", "L n_samples", [&](size_t r) {
        p.J = dalloc<double>(s, r); p.w = dalloc<double>(s, r); }))
    return rc;
  if (int rc = grow(s, who, s->plan_l_pool, l1, 4 * (2 * nu + nr) + 24, "means and references", "L (T + 1)", [&](size_t r) {
        p.mean = dalloc<float>(s, r * nu); p.xref = dalloc<float>(s, r * nr); p.uref = dalloc<float>(s, r * nu);
        p.seed = dalloc<unsigned>(s, r); p.wsum = dalloc<double>(s, r); p.sel = dalloc<int>(s, r); p.status = dalloc<int>(s, r); }))
    return rc;
  if (int rc = grow(s, who, s->plan_h_pool, (size_t)L * n_iter, 16, "cost record", "L n_iter", [&](size_t r) { p.hist = dalloc<double>(s, 2 * r); }))
    return rc;
  if (copy_async(s, p.mean, mean, 4 * lt * nu) != 0 || copy_async(s, (void*)p.xref, xref, 4 * l1 * nr) != 0 ||
      (uref && copy_async(s, (void*)p.uref, uref, 4 * lt * nu) != 0) || copy_async(s, (void*)p.seed, seeds, 4 * (size_t)L) != 0) return -2;
  DevPlan q = p;
  q.L = L; q.T = T; q.n_iter = n_iter;
  if (!uref) q.uref = nullptr;
  DevRoll& r = s->plan_roll;
  r = DevRoll{};
  r.n = (int)n; r.T = T; r.nsub = n_substeps; r.ctrl = p.ctrl;
  const int* fan;                              // the fan-out list, uploaded once: no host copy inside the iterations
  if (int rc = fan_out_ids(s, slots, L, K, &fan)) return rc;
  for (int it = 0; it < n_iter; it++) {        // no host synchronisation inside the iterations
    q.iter = it;
    warp_launch(s, "plan_sample", (int)n, 0, PlanWarp<0>{s->m, s->d, q});
    launch_state<true>(s, nullptr, fan, N);      // the state bank's fan-out (fd_fan_out with K columns)
    launch_step1(s);                           // what the rows do not carry, as fb_rollout runs it
    q.t = -1;
    warp_launch(s, "plan_cost", (int)n, 0, PlanWarp<1>{s->m, s->d, q});
    for (int t = 0; t < T; t++) {
      r.t = q.t = t;
      warp_launch(s, "rollout_input", N, 0, RollInput{s->m, s->d, r, nullptr});
      step_run(s, n_substeps);                 // fb_step's launches (the step graph)
      warp_launch(s, "plan_cost", (int)n, 0, PlanWarp<1>{s->m, s->d, q});
    }
    warp_launch(s, "plan_weights", L, 0, PlanWarp<2>{s->m, s->d, q});
    warp_launch(s, "plan_update", L * ((T + PLAN_STEPS - 1) / PLAN_STEPS), 0, PlanWarp<3>{s->m, s->d, q});
  }
  if (launch_check(s, who) != 0) return -2;
  p.L = L; p.T = T; p.n_iter = n_iter;
  s->plan_done = L;
  return sync_stream(s);                       // host inputs may be reused once the call returns
}

int fb_plan_read(FbHandle s, float* mean, double* cost, double* sample_cost, float* samples, int32_t* status, int is_device) {
  if (!s) return -1;
  if (s->plan_done < 1) { s->err = "fb_plan_read: no plan to read (fb_plan)"; return -1; }
  const DevPlan& p = s->plan;
  const size_t L = p.L, n = L * p.K, nu = s->m.nu;
  return read_out(s, {{mean, p.mean, 0, 4 * L * p.T * nu, 1}, {cost, p.hist, 0, 16 * L * p.n_iter, 1}, {sample_cost, p.J, 0, 8 * n, 1},
                      {samples, p.ctrl, 0, 4 * n * p.T * nu, 1}, {status, p.status, 0, 4 * L, 1}});
}

}  // extern "C"

// -------------------------------------------------------------------------------------------
// system identification (fb_sid_accumulate; fb_sid.h): its own kernel parameter (DevSid) and buffers, reading the outputs of the last
// parameter-Jacobian query in place
template <int KIND> struct SidWarp {
  DevModel m; DevData d; DevSid p;
  FB_DEVM void operator()(unsigned char*, int w) const { if (KIND == 0) ksid_resid(m, d, p, w); else ksid_sum(p, w); }
};

extern "C" {

int fb_sid_accumulate(FbHandle s, int query, int L, const int32_t* problem, int n, const float* target, const double* weight,
                      const float* sample_weight, int reset, int is_device) {
  if (!s) return -1;
  const char* who = "fb_sid_accumulate";
  if (query != FB_SID_TRANSITION && query != FB_SID_INVERSE) { s->err = "fb_sid_accumulate: query is FB_SID_TRANSITION or FB_SID_INVERSE"; return -1; }
  const bool inv = query == FB_SID_INVERSE;
  const FdQuery& q = inv ? s->fd_pinv : s->fd_ptr;
  if (q.done < 1) { s->err = std::string(who) + ": no parameter Jacobians to accumulate (" + q.name + ")"; return -1; }
  if (s->launches != q.at) {
    s->err = std::string(who) + ": the handle launched kernels since the last " + q.name + ", so its outputs and its nominal envs' flags are no longer that call's";
    return -1; }
  if (n != q.done) { s->err = std::string(who) + ": n = " + std::to_string(n) + " against the " + std::to_string(q.done) + " problems of the last " + q.name; return -1; }
  const DevModel& m = s->m;
  const int k = q.p.nin, rows = inv ? m.nv : 2 * m.nv + m.na, nr = inv ? m.nv : m.nq + m.nv + m.na;
  if (L < 1) { s->err = "fb_sid_accumulate: L >= 1 fit problems"; return -1; }
  if (!reset && (L != s->sid_L || k != s->sid_k)) {
    s->err = s->sid_L < 1 ? std::string(who) + ": no sums to add to (reset = 1 starts them)" :
             std::string(who) + ": without reset, L and k must be the sums' (L = " + std::to_string(s->sid_L) + ", k = " + std::to_string(s->sid_k) + ")";
    return -1; }
  if (!problem || !weight) { s->err = "fb_sid_accumulate: problem and weight must not be NULL"; return -1; }
  if (!inv && !target) { s->err = "fb_sid_accumulate: a transition residual needs its target x'_obs"; return -1; }
  std::vector<int> ptr(L + 1, 0), order;
  for (int i = 0; i < n; i++) {
    if (problem[i] < -1 || problem[i] >= L) {
      s->err = std::string(who) + ": problem[" + std::to_string(i) + "] = " + std::to_string(problem[i]) + " is not in [-1, L)"; return -1; }
    if (problem[i] >= 0) ptr[problem[i] + 1]++;
  }
  for (int l = 0; l < L; l++) ptr[l + 1] += ptr[l];
  order.resize(ptr[L]);
  { std::vector<int> at(ptr.begin(), ptr.end() - 1); for (int i = 0; i < n; i++) if (problem[i] >= 0) order[at[problem[i]]++] = i; }
  for (int c = 0; c < rows; c++)
    if (!(weight[c] >= 0.0) || !std::isfinite(weight[c])) { s->err = "fb_sid_accumulate: the weights must be >= 0 and finite"; return -1; }
  if (!is_device) {
    if (sample_weight) for (int i = 0; i < n; i++)
      if (!(sample_weight[i] >= 0.0f) || !std::isfinite(sample_weight[i])) { s->err = "fb_sid_accumulate: the sample weights must be >= 0 and finite"; return -1; }
    if (target && !all_finite(target, (size_t)n * nr)) { s->err = "fb_sid_accumulate: non-finite target"; return -1; }
  }
  dev_select(s);
  DevSid& p = s->sid;
  if (reset) s->sid_L = 0;                     // (growing the sums drops them)
  if (int rc = grow(s, who, s->sid_t_pool, (size_t)n, 8 * (size_t)(2 * m.nv + m.na + 1) + 4 * (size_t)(m.nq + m.nv + m.na + 3),
                    "transition scratch", "n", [&](size_t r) {
        p.res = dalloc<double>(s, r * (2 * m.nv + m.na)); p.tcost = dalloc<double>(s, r); p.tbad = dalloc<int>(s, r);
        p.target = dalloc<float>(s, r * (m.nq + m.nv + m.na)); p.sw = dalloc<float>(s, r); p.order = dalloc<int>(s, r);
        p.W = dalloc<double>(s, 2 * m.nv + m.na); }))
    return rc;
  const size_t E = (size_t)k * k + k + 1;
  if (int rc = grow(s, who, s->sid_s_pool, (size_t)L * E, 8, "sums", "L (k^2 + k + 1)", [&](size_t r) { p.H = dalloc<double>(s, r); }))
    return rc;
  if (int rc = grow(s, who, s->sid_l_pool, (size_t)L + 1, 12, "per-problem words", "L + 1", [&](size_t r) {
        p.count = dalloc<int>(s, r); p.bad = dalloc<int>(s, r); p.ptr = dalloc<int>(s, r); }))
    return rc;
  if (copy_async(s, (void*)p.order, order.data(), 4 * order.size()) != 0 || copy_async(s, (void*)p.ptr, ptr.data(), 4 * (size_t)(L + 1)) != 0 ||
      copy_async(s, (void*)p.W, weight, 8 * (size_t)rows) != 0 || (target && copy_async(s, (void*)p.target, target, 4 * (size_t)n * nr) != 0) ||
      (sample_weight && copy_async(s, (void*)p.sw, sample_weight, 4 * (size_t)n) != 0)) return -2;
  DevSid c = p;
  c.L = L; c.k = k; c.rows = rows; c.nr = nr; c.ncol = q.p.ncol; c.inverse = inv; c.reset = reset != 0;
  c.J = q.p.blk[0].out; c.pred = q.p.nom[0].out;
  if (!target) c.target = nullptr;
  if (!sample_weight) c.sw = nullptr;
  c.g = p.H + (size_t)L * k * k; c.cost = c.g + (size_t)L * k;      // the sums' layout: H, g, cost
  if (ptr[L] > 0) warp_launch(s, "sid_resid", ptr[L], 0, SidWarp<0>{s->m, s->d, c});
  warp_launch(s, "sid_sum", L * (k * (k + 1) / 2 + k + 1), 0, SidWarp<1>{s->m, s->d, c});
  if (launch_check(s, who) != 0) return -2;
  s->sid_L = L; s->sid_k = k;
  return sync_stream(s);                       // host inputs may be reused once the call returns
}

int fb_sid_read(FbHandle s, double* H, double* g, double* cost, int32_t* count, int32_t* bad, int is_device) {
  if (!s) return -1;
  if (s->sid_L < 1) { s->err = "fb_sid_read: no sums to read (fb_sid_accumulate)"; return -1; }
  const DevSid& p = s->sid;
  const size_t L = s->sid_L, k = s->sid_k;
  const double *pg = p.H + L * k * k, *pc = pg + L * k;      // (the sums' layout: H, g, cost)
  return read_out(s, {{H, p.H, 0, 8 * L * k * k, 1}, {g, pg, 0, 8 * L * k, 1}, {cost, pc, 0, 8 * L, 1}, {count, p.count, 0, 4 * L, 1},
                      {bad, p.bad, 0, 4 * L, 1}});
}

}  // extern "C"
