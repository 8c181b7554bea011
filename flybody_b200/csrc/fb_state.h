// fb_state.h -- compact per-env state rows (fb_state_save / fb_state_load): what physics.get_state() / physics.set_state() are
// to a single MuJoCo model, for the envs of a batch and with the task's own per-env state.
//
// A row holds what the next control step reads and the position / velocity stage does not rewrite: the integrated state, the
// solver's warm start, the sensor sums, the rows a caller reads between steps and the device task's per-env arrays.  The host
// lays the row out as a table of segments (flybody_b200.cu: state_layout); a segment is n 4-byte slots found `stride` slots
// apart from env to env -- a field of the record (stride = the record stride) or a compact per-env array (stride = its row).
// Segments start on 16-byte boundaries of the row and rows are whole 16-byte units, so a segment whose source is aligned as
// well moves in 128-bit accesses.  One warp moves one (env, slot) pair, lanes striding over each segment.
#pragma once
#include "fb_task.h"

struct StSeg { void* base; unsigned stride; int n, off, vec /* source rows 16-byte aligned */, bytes /* one unsigned char per env, kept in one slot */; };
struct StArgs {
  const StSeg* segs; int nseg;
  unsigned* bank; unsigned row;              // [n_slots][row]
  const int *env, *slot; int n;              // the pairs of the call; nullptr: the identity (pair w = env w, slot w)
  const DevTask* task;                       // FB_TASK_VISION: a load brings the env's terrain along
};
#ifdef __CUDACC__
typedef uint4 St4;
#else
struct alignas(16) St4 { unsigned x, y, z, w; };
#endif

template <bool LOAD> FB_DEV void kstate_copy(const StArgs& a, int w, int y) {
  const int e = a.env ? a.env[w] : w, slot = a.slot ? a.slot[w] : w;
  unsigned* row = a.bank + (size_t)slot * a.row;
  for (int k = 0; k < a.nseg; k++) {
    const StSeg& g = a.segs[k];
    unsigned* r = row + g.off;
    if (g.bytes) {
      unsigned char* p = (unsigned char*)g.base + e;
      if (y == 0) { if (LOAD) *p = (unsigned char)r[0]; else r[0] = *p; }
      continue;
    }
    unsigned* p = (unsigned*)g.base + (size_t)e * g.stride;
    const int n4 = g.vec ? g.n >> 2 : 0;
    for (int i = y; i < n4; i += FB_NY) { if (LOAD) ((St4*)p)[i] = ((const St4*)r)[i]; else ((St4*)r)[i] = ((const St4*)p)[i]; }
    for (int i = 4 * n4 + y; i < g.n; i += FB_NY) { if (LOAD) p[i] = r[i]; else r[i] = p[i]; }
  }
}
// vision task: the loaded row names another terrain of the bank than the env holds -> copy it, as the env's reset would
FB_DEV void kstate_terrain(const StArgs& a, int w, int y, int old_pick) {
  if (!a.task || a.task->kind != FB_TASK_VISION) return;
  const int e = a.env ? a.env[w] : w, pick = a.task->pick[e];
  if (pick == old_pick || pick < 0 || pick >= a.task->n_bank) return;
  tk_terrain_copy(*a.task, e, y, pick);
}
FB_DEV int kstate_pick(const StArgs& a, int w) { return (a.task && a.task->kind == FB_TASK_VISION) ? a.task->pick[a.env ? a.env[w] : w] : -1; }
