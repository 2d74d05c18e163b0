// Wavefront kernels: CVP (per-cluster batches, whole-grid single plan, epilogue) and Dijkstra on the band engine.
// (part of libmeshnav_b200.so: included by meshnav.cu, which holds the C ABI and all host code)
#pragma once
#include "launch.cuh"
#include "problems.cuh"

using namespace mnb;

// ============================================================================
// wavefront kernels
// ============================================================================
// round watchdog (group-uniform): far above the dependency depth of any sane mesh (a grid needs ~ D/h rounds),
// small enough that a livelock is reported in seconds instead of hanging the device
static inline uint32_t watchdog_rounds(uint32_t V) { return 200000u + 256u * (uint32_t)sqrt((double)V); }

struct WaveWorkspace {     // per group (index g): state + g*V etc.
  uint4* state;
  uint32_t* ext;     // level-2 ids / level-pool references of flagged labels (band_engine.cuh)
  uint32_t* root;    // cascade roots of flagged labels
  uint32_t* pool;    // level pool: records of pop times with more than 3 cascade levels, pool_cap words per group
  uint32_t pool_cap;
  uint32_t* last_eval; uint32_t* dirty;   // inflation only (V entries): clean-candidate stamps (InflationProblem)
  uint4* skipw;      // clean-candidate words of the batch round loop (batch_engine.cuh)
  uint32_t* chg;
  uint32_t* ver;     // single-plan only (V entries): input versions for the in-round sweeps
  uint32_t* mark;
  uint32_t* list0;
  uint32_t* list1;
  GroupCtl* ctl;
};

struct CvpKernelArgs {
  uint32_t V;
  const float* pos;
  const uint32_t* faces;
  const uint32_t* cor_ptr; const int4* cor_idx; const float4* cor_w;
  const int4* ell_idx; const float4* ell_w; const double4* ell_geo;
  const float* cost; const uint8_t* invalid;
  WaveWorkspace ws;
  uint32_t n_queries;
  const uint32_t* seed_faces;   // [n_queries] device
  const float* seed_pos;        // [3 n_queries] device
  long long robot_face;         // single query only, -1 = none
  double cost_limit, goal_dist_offset;
  float delta;
  float* out_dist;              // [n_queries][V]
  uint32_t* out_pred;           // single query or null
  float* out_dir;
  int32_t* out_cut;
  unsigned int* next_query;
  const int* cancel_flag;
  uint32_t max_rounds;
  int sweeps;                   // in-round sweeps of a single plan (0 = off, -1 = from the band width)
  float hop;                    // ~ one dependency hop in potential units (1.35 x mean edge weight)
  uint32_t slots;               // k_cvp_grid: GridStage slots per CTA (in the tail padding: the struct keeps its size)
};
// the arguments of the matrix form of k_cvp_batch.  A type of its own rather than a field of CvpKernelArgs: the batch
// kernels pass their arguments by reference to out-of-line functions, which copy them to the stack, so a larger
// CvpKernelArgs would grow the stack frame of every CVP batch kernel.
struct CvpMatrixArgs : CvpKernelArgs {
  TargetSet tg;
};

template <int CS>
__device__ __forceinline__ void group_coords(uint32_t& g, uint32_t& gthreads, uint32_t& gtid) {
  if constexpr (CS == 0) {
    g = 0; gthreads = gridDim.x * blockDim.x; gtid = blockIdx.x * blockDim.x + threadIdx.x;
  } else {
    g = blockIdx.x / CS; gthreads = CS * blockDim.x; gtid = (blockIdx.x % CS) * blockDim.x + threadIdx.x;
  }
}

__device__ __forceinline__ void ctl_reset(GroupCtl* ctl, unsigned int n0, float seed_min) {
  ctl->count[0] = n0; ctl->count[1] = 0; ctl->count[2] = 0;
  ctl->m_tau[0] = INF_BITS; ctl->m_tau[1] = INF_BITS; ctl->m_tau[2] = 0u;
  ctl->lo[0] = INF_BITS; ctl->lo[1] = INF_BITS; ctl->lo[2] = __float_as_uint(seed_min);
  ctl->goal_ring[0] = INF_BITS; ctl->goal_ring[1] = INF_BITS; ctl->stop_ring[0] = 0; ctl->stop_ring[1] = 0;
  ctl->goal_bits = INF_BITS; ctl->robot_left = 0;
  time_put(ctl->goal_time, ev_normal(__uint_as_float(INF_BITS), 0u));
  ctl->pool_top = 0u;
  ctl->done_ring[0] = 0u; ctl->done_ring[1] = 0u;
}

// the label of a seed with potential d (its pop time is (d, seed)): the engine's 16-byte word or the lean float label
__device__ __forceinline__ void put_seed_label(uint4& w, float d) { w = make_uint4(__float_as_uint(d), __float_as_uint(d), 0u, 0u); }
__device__ __forceinline__ void put_seed_label(float& w, float d) { w = d; }

// The seeding of a fresh wave (one thread): the n seeds s[k] take their labels d[k] and are fixed, their eligible
// neighbours are the first candidates in list 0, and the control block is reset with the band at lo_init.
template <class P>
__device__ __forceinline__ void seed_wave(const P& prob, GroupCtl* ctl, uint32_t* mark, uint32_t* list0, const uint32_t* s, const float* d,
                                          int n, float lo_init) {
  for (int k = 0; k < n; ++k) { put_seed_label(prob.state[s[k]], d[k]); mark[s[k]] = MARK_FIXED; }
  unsigned int n0 = 0;
  for (int k = 0; k < n; ++k)
    prob.activate(s[k], [&](uint32_t x) {
      if (mark[x] == MARK_NONE && prob.eligible(x)) { mark[x] = MARK_CAND; list0[n0++] = x; }
    });
  ctl_reset(ctl, n0, lo_init);
}

// The fields every CvpProblem sets: the mesh tables, costs, gates and cost limit of a; the label store of one workspace
// group (its labels, side arrays, level pool and control block); the seed face; the goal cutoff's pop time (+inf: not
// armed); the outputs (any may be null).  No in-round sweeps (ver), strict rule off.
__device__ __forceinline__ void cvp_problem(const CvpKernelArgs& a, uint4* state, uint32_t* ext, uint32_t* root, uint32_t* chg, uint32_t* pool,
                                            uint32_t pool_cap, GroupCtl* ctl, const SeedFace& sd, const EvTime& goal_t, uint32_t* pred, float* dir, int32_t* cut,
                                            CvpProblem& prob) {
  prob.cor_ptr = a.cor_ptr; prob.cor_idx = a.cor_idx; prob.cor_w = a.cor_w; prob.cost = a.cost; prob.invalid = a.invalid; prob.cost_limit = a.cost_limit;
  prob.state = state; prob.ext_arr = ext; prob.root_arr = root; prob.chg = chg;
  prob.pool_w = pool; prob.pool = pool; prob.pool_cap = pool_cap; prob.pool_top = &ctl->pool_top; prob.pool_overflow = &ctl->pool_overflow;
  prob.s0 = sd.s[0]; prob.s1 = sd.s[1]; prob.s2 = sd.s[2]; prob.seed_noexpand = sd.noexpand; prob.seed_max_d = sd.seed_max;
  prob.goal_t = goal_t; prob.pred = pred; prob.dir = dir; prob.cut = cut;
  prob.ver = nullptr; prob.deferred_m = __uint_as_float(INF_BITS); prob.strict = 0;
}
// ... and the ELL tables of the 8-lane form (no outputs: the wavefront writes labels only)
__device__ __forceinline__ void cvp_ell_problem(const CvpKernelArgs& a, uint4* state, uint32_t* ext, uint32_t* root, uint32_t* chg, uint32_t* pool,
                                                uint32_t pool_cap, GroupCtl* ctl, const SeedFace& sd, const EvTime& goal_t, bool prefetch_marks, CvpEllProblem& prob) {
  cvp_problem(a, state, ext, root, chg, pool, pool_cap, ctl, sd, goal_t, nullptr, nullptr, nullptr, prob);
  prob.ell_idx = a.ell_idx; prob.ell_w = a.ell_w; prob.ell_geo = a.ell_geo; prob.prefetch_marks = prefetch_marks;
}

// Matrix form, after the seeding (and a group barrier): ctl->targets_left = tg.distinct less the targets that are done
// before the first round -- a seed (MARK_FIXED: its label is final) or a vertex that never becomes a candidate
// (eligible(v) false: its entry stays +inf).  If none is left the flag of round 0 is raised and the wave runs no round.
// Called by every thread of the group; a group barrier must follow.
template <class Eligible>
__device__ __forceinline__ void count_targets_done_at_init(const TargetSet& tg, GroupCtl* ctl, const uint32_t* mark, uint32_t V,
                                                           uint32_t gthreads, uint32_t gtid, Eligible eligible) {
  unsigned int done = 0;
  for (uint32_t w = gtid; w <= (V >> 5); w += gthreads) {
    uint32_t b = __ldg(&tg.bits[w]);
    while (b) {
      const uint32_t v = (w << 5) + (uint32_t)(__ffs(b) - 1);
      b &= b - 1u;
      if (__ldcg(&mark[v]) == MARK_FIXED || !eligible(v)) done++;
    }
  }
  done = __reduce_add_sync(0xffffffffu, done);
  if ((threadIdx.x & 31) == 0 && done && atomicSub(&ctl->targets_left, (int)done) == (int)done) atomicOr(&ctl->done_ring[0], 1u);
}

#include "batch_engine.cuh"

#ifndef MNB_CVP_MINBLOCKS
#define MNB_CVP_MINBLOCKS 1
#endif
#ifndef MNB_CVP_THREADS
#define MNB_CVP_THREADS 512
#endif
// The prologue of a single-plan CVP wave (k_cvp, k_cvp_grid): the clearing pass (the sweep versions only for the kernel
// with in-round sweeps), the problem, and -- unless RESUME -- the seeding; then the robot face's vertices rv (none:
// 0xffffffff) and how many of them are not fixed.  If none is left, the robot face is the seed face and the cutoff is armed
// when the last seed pops (cvp:763-771).  Called by every thread of the group; ends with a group barrier.
template <int CS, bool RESUME>
__device__ __forceinline__ void cvp_single_setup(const CvpKernelArgs& a, bool clear_ver, bool prefetch_marks, uint32_t gthreads, uint32_t gtid,
                                                 CvpEllProblem& prob, uint32_t (&rv)[3]) {
  uint4* state = a.ws.state; uint32_t* mark = a.ws.mark; GroupCtl* ctl = a.ws.ctl;
  if constexpr (!RESUME) {
    for (uint32_t v = gtid; v < a.V; v += gthreads) {
      state[v] = state_inf(); mark[v] = MARK_NONE; a.ws.chg[v] = 0u;
      if (clear_ver) a.ws.ver[v] = 0u;
    }
    group_sync<CS>();
  }
  const CvpSeeds sd = cvp_seeds(a.faces, a.pos, a.cost, a.invalid, a.cost_limit, a.seed_faces[0], a.seed_pos);
  cvp_ell_problem(a, state, a.ws.ext, a.ws.root, a.ws.chg, a.ws.pool, a.ws.pool_cap, ctl, sd, ev_normal(__uint_as_float(INF_BITS), 0u), prefetch_marks, prob);
  prob.ver = a.ws.ver;
  const bool has_robot = a.robot_face >= 0;
  for (int k = 0; k < 3; ++k) rv[k] = has_robot ? a.faces[3 * (size_t)a.robot_face + k] : 0xffffffffu;
  if (gtid == 0) {
    if constexpr (!RESUME) seed_wave(prob, ctl, mark, a.ws.list0, sd.s, sd.d, 3, sd.seed_min);
    if (has_robot) {
      int left = 0;
      for (int k = 0; k < 3; ++k) if (mark[rv[k]] != MARK_FIXED) left++;
      ctl->robot_left = left;
      if (left == 0) {
        ctl->goal_ring[0] = __float_as_uint((float)((double)sd.seed_max + a.goal_dist_offset));
        uint32_t sl = sd.s[0]; float sdl = sd.d[0];
        for (int k = 1; k < 3; ++k) if (sd.d[k] > sdl || (sd.d[k] == sdl && sd.s[k] > sl)) { sl = sd.s[k]; sdl = sd.d[k]; }
        time_put(ctl->goal_time, ev_normal(sdl, sl));
      }
    }
  }
  group_sync<CS>();
}

// A single plan on one cluster of CS CTAs (mnb_set_tuning(cluster >= 1)).
// RESUME (mnb_cvp_replan): the workspace holds a rolled-back wave (k_replan_rollback, k_replan_frontier), so the clearing
// pass and the seeding are skipped and the band starts at T0 (DESIGN §4, "Replan").
template <int CS, bool RESUME = false>
__global__ void __launch_bounds__(MNB_CVP_THREADS, MNB_CVP_MINBLOCKS) k_cvp(const CvpKernelArgs a) {
  __shared__ Stage st;
  uint32_t g, gthreads, gtid;
  group_coords<CS>(g, gthreads, gtid);
  GroupCtl* ctl = a.ws.ctl;
  if (threadIdx.x == 0) stage_init(st);
  __syncthreads();
  CvpEllProblem prob;
  uint32_t rv[3];
  cvp_single_setup<CS, RESUME>(a, false, false, gthreads, gtid, prob, rv);
  const int has_robot = a.robot_face >= 0;
  float delta = a.delta;
  if (has_robot && a.goal_dist_offset < (double)delta) delta = (float)fmax(a.goal_dist_offset, 1e-4);
  // a resumed band starts at T0: every kept label (and seed) lies below it (k_replan_rollback set lo[2] = T0's key)
  const float band_init = RESUME ? __uint_as_float(__ldcg(&ctl->lo[2])) : prob.seed_max_d;
  run_band_rounds_sub8<CS, false, CvpEllProblem, RESUME>(prob, ctl, a.ws.list0, a.ws.list1, a.ws.mark, st, delta, gthreads, gtid, has_robot,
                        rv[0], rv[1], rv[2], a.goal_dist_offset, a.cancel_flag, nextafterf(band_init, __uint_as_float(INF_BITS)),
                        a.max_rounds, 0, a.V);     // in-round sweeps are compiled into the whole-grid kernel only
  group_sync<CS>();
  if (a.out_dist)
    for (uint32_t v = gtid; v < a.V; v += gthreads) a.out_dist[v] = __uint_as_float(a.ws.state[v].x);
}

// Batches of full-field plans (mnb_cvp_batch): the lean round loop of batch_engine.cuh.  One wavefront per CTA (CS = 1) or
// per cluster of CS CTAs; persistent groups pull goal indices from an atomic counter.
#ifndef MNB_BATCH_THREADS
#define MNB_BATCH_THREADS 256
#endif
#ifndef MNB_BATCH_MINBLOCKS
#define MNB_BATCH_MINBLOCKS 4
#endif

// The CVP epilogue: predecessors_ / direction_ / cutting_faces_ (cvp:423-431,493-517) from the FINAL labels of a wavefront.
// Every vertex replays its faces once more in event order and evaluates the winning face with the literal acos form.  Done
// after the wavefront so that the stored angles use the final source potentials.  Run by k_cvp_epilogue for a single plan
// and by k_cvp_batch<CS, true> for each goal of a batch, on the wavefront's own workspace group.
// The problem object: the workspace group's labels, the goal's seed face sf (seed point sp), the goal cutoff's pop time (not
// armed: +inf) and the outputs (any may be null).
__device__ __forceinline__ void cvp_epilogue_problem(const CvpKernelArgs& a, uint4* state, uint32_t* ext, uint32_t* root, uint32_t* chg,
                                                     uint32_t* pool, GroupCtl* ctl, uint32_t sf, const float* sp, const EvTime& goal_t,
                                                     uint32_t* pred, float* dir, int32_t* cut, CvpProblem& prob) {
  SeedFace sd = cvp_seeds(a.faces, a.pos, a.cost, a.invalid, a.cost_limit, sf, sp);
  sd.seed_max = __builtin_huge_valf();       // final labels: the replay tests every source for a seed
  cvp_problem(a, state, ext, root, chg, pool, a.ws.pool_cap, ctl, sd, goal_t, pred, dir, cut, prob);
}

// one vertex c of the epilogue (goal: the goal cutoff's potential, +inf when not armed).  ROW: the replay runs on c's ELL
// row in registers (CvpProblem::replay_row), and a vertex it does not cover (more than 8 faces, a cascade member among the
// sources) is handed to csr(c), which runs CvpProblem::epilogue_csr -- at once or in a launch of its own.  !ROW: the CSR
// replay in line, for a caller whose registers cannot hold a row: at the 64 registers of the batch kernels the row
// replay spills, and the batch with fields was measured 13 % slower with it.  ALL_CSR (with ROW; a test hook): every vertex
// the row replay would take is handed to csr(c) instead, so that the two replays can be compared on the same labels.
template <bool ROW, bool ALL_CSR = false, class Csr>
__device__ __forceinline__ void cvp_epilogue_vertex(CvpProblem& prob, const int4* __restrict__ ell_idx, const float4* __restrict__ ell_w,
                                                    GroupCtl* ctl, uint32_t sf, float goal, uint32_t c, Csr csr) {
  const int4* row = ell_idx + (size_t)c * ELL_W;
  int4 ix[ELL_W];                                        // (requested together with the label of c)
  if constexpr (ROW && !ALL_CSR) {
#pragma unroll
    for (int j = 0; j < (int)ELL_W; ++j) ix[j] = __ldg(&row[j]);
  }
  const uint4 lw = __ldcg(&prob.state[c]);
  const float d = __uint_as_float(lw.x);
  // statistic: labels whose pop time has more than 3 cascade levels (their tails live in the level pool; exact)
  if (__float_as_uint(d) != INF_BITS && (lw.w >> 31) && (__ldcg(&prob.ext_arr[c]) & EXT_POOL)) atomicAdd(&ctl->deep_labels, 1u);
  if (prob.seed_index(c) >= 0) {                         // cvp:719-728
    if (prob.pred) prob.pred[c] = c;
    if (prob.dir) prob.dir[c] = 0.0f;
    if (prob.cut) prob.cut[c] = (int32_t)sf;
    return;
  }
  if constexpr (!ROW) {
    int win = -1; float nd, wu1 = 0, wu2 = 0; EvFull nt;
    if (__float_as_uint(d) != INF_BITS && prob.eligible(c))
      prob.replay(c, __uint_as_float(INF_BITS), goal, 0xfffffff0u /* final labels: nothing is deferred */, nd, nt, win, wu1, wu2);
    prob.write_aux(c, win, wu1, wu2);
  } else {
    if (__float_as_uint(d) == INF_BITS || !prob.eligible(c)) { prob.write_aux_none(c); return; }
    int win; float4 ww; float wu1, wu2;
    if (ALL_CSR || !prob.replay_row(c, ix, ell_w, __uint_as_float(INF_BITS), goal, 0xfffffff0u /* final labels: nothing is deferred */, win, ww, wu1, wu2)) {
      csr(c);
      return;
    }
    if (win < 0) prob.write_aux_none(c);
    else prob.write_aux(c, __ldg(&row[win]), ww, wu1, wu2);
  }
}

// k_cvp_batch<CS, true>: the epilogue of goal q over the group's workspace, rows q of out_pred / out_dir / out_cut (each may
// be null).  Out of line: its frame (the replay holds a vertex's faces) does not weigh on the registers of the round loop.
__device__ __noinline__ void batch_fields_epilogue(const CvpKernelArgs& a, const BatchGroup& G, uint32_t q, uint32_t gthreads, uint32_t gtid) {
  const uint32_t V = a.V;
  const size_t row = (size_t)q * V;
  const uint32_t sf = a.seed_faces[q];
  CvpProblem prob;
  cvp_epilogue_problem(a, G.state, G.ext_arr, G.root_arr, G.chg, G.pool, G.ctl, sf, a.seed_pos + 3 * (size_t)q, ev_normal(__uint_as_float(INF_BITS), 0u),
                       a.out_pred ? a.out_pred + row : nullptr, a.out_dir ? a.out_dir + row : nullptr, a.out_cut ? a.out_cut + row : nullptr, prob);
  for (uint32_t v = gtid; v < V; v += gthreads) cvp_epilogue_vertex<false>(prob, a.ell_idx, a.ell_w, G.ctl, sf, __uint_as_float(INF_BITS), v, [](uint32_t) {});
}

// FIELDS = false: potentials only (mnb_cvp_batch, and mnb_cvp_batch_fields asked for potentials alone).  FIELDS = true:
// each group also runs the epilogue of its goal before it takes the next one, and takes none once the cancel flag is set.
// Args = CvpMatrixArgs (with FIELDS = false; mnb_cvp_matrix): the matrix form.  A wave ends once the target vertices of
// a.tg have settled and writes their potentials, row q of a.tg.out, instead of the V-sized row; no new goal is taken once
// the cancel flag is set.
template <int CS, bool FIELDS, class Args = CvpKernelArgs>
__global__ void __launch_bounds__(MNB_BATCH_THREADS, MNB_BATCH_MINBLOCKS) k_cvp_batch(const Args a) {
  constexpr bool MATRIX = std::is_same_v<Args, CvpMatrixArgs>;
  static_assert(!(FIELDS && MATRIX), "the matrix form writes potentials only");
  __shared__ BatchStage st;
  __shared__ BatchWork wk;
  uint32_t g, gthreads, gtid;
  group_coords<CS>(g, gthreads, gtid);
  const uint32_t V = a.V;
  BatchGroup G;
  G.state = a.ws.state + (size_t)g * V; G.root_arr = a.ws.root + (size_t)g * V; G.ext_arr = a.ws.ext + (size_t)g * V;
  G.chg = a.ws.chg + (size_t)g * V; G.mark = a.ws.mark + (size_t)g * V; G.pool = a.ws.pool + (size_t)g * a.ws.pool_cap;
  G.pool_cap = a.ws.pool_cap; G.ctl = a.ws.ctl + g; G.skipw = a.ws.skipw + (size_t)g * V;
  uint32_t* list0 = a.ws.list0 + (size_t)g * V;
  uint32_t* list1 = a.ws.list1 + (size_t)g * V;
  GroupCtl* ctl = G.ctl;
  if (threadIdx.x == 0) { stage_init(st); wk.n = 0; wk.ns = 0; }
  __syncthreads();
  for (;;) {
    if (gtid == 0) {
      if constexpr (FIELDS || MATRIX) ctl->query = (a.cancel_flag && *(const volatile int*)a.cancel_flag) ? a.n_queries : atomicAdd(a.next_query, 1u);
      else ctl->query = atomicAdd(a.next_query, 1u);
    }
    group_sync<CS>();
    const uint32_t q = __ldcg(&ctl->query);
    if (q >= a.n_queries) break;
    for (uint32_t v = gtid; v < V; v += gthreads) { G.state[v] = state_inf(); G.mark[v] = MARK_NONE; G.chg[v] = 0u; G.skipw[v] = make_uint4(INF_BITS, INF_BITS, 0u, 0u); }
    group_sync<CS>();
    const CvpSeeds cs = cvp_seeds(a.faces, a.pos, a.cost, a.invalid, a.cost_limit, a.seed_faces[q], a.seed_pos + 3 * (size_t)q);
    const SeedFace sd = cs;
    if (gtid == 0) {
      for (int k = 0; k < 3; ++k) { put_seed_label(G.state[cs.s[k]], cs.d[k]); G.mark[cs.s[k]] = MARK_FIXED; }
      unsigned int n0 = 0;
      for (int k = 0; k < 3; ++k) {
        const uint32_t kb = a.cor_ptr[cs.s[k]], ke = a.cor_ptr[cs.s[k] + 1];
        for (uint32_t kk = kb; kk < ke; ++kk) {
          const int4 ix = a.cor_idx[kk];
          const uint32_t xs[2] = {(uint32_t)ix.x, (uint32_t)ix.y};
          for (int t = 0; t < 2; ++t) {
            const uint32_t x = xs[t];
            // (CvpProblem::eligible written out: through the call k_cvp_batch<1, false> takes 16 bytes more stack)
            if (G.mark[x] == MARK_NONE && !(a.invalid && a.invalid[x]) && !((double)a.cost[x] >= a.cost_limit)) { G.mark[x] = MARK_CAND; list0[n0++] = x; }
          }
        }
      }
      ctl_reset(ctl, n0, cs.seed_min);
      if constexpr (MATRIX) ctl->targets_left = (int)a.tg.distinct;
    }
    group_sync<CS>();
    if constexpr (MATRIX) {
      count_targets_done_at_init(a.tg, ctl, G.mark, V, gthreads, gtid,
                                 [&](uint32_t v) { return CvpProblem::eligible(v, a.cost, a.invalid, a.cost_limit); });
      group_sync<CS>();
    }
    run_band_rounds_batch<CS, MATRIX>(a, G, list0, list1, st, wk, a.delta, gthreads, gtid, sd, nextafterf(sd.seed_max, __uint_as_float(INF_BITS)));
    group_sync<CS>();
    if constexpr (MATRIX) {
      float* om = a.tg.out + (size_t)q * a.tg.m;
      for (uint32_t j = gtid; j < a.tg.m; j += gthreads) om[j] = __uint_as_float(__ldcg(&G.state[a.tg.list[j]]).x);
    } else if (a.out_dist) {
      float* od = a.out_dist + (size_t)q * V;
      for (uint32_t v = gtid; v < V; v += gthreads) od[v] = __uint_as_float(__ldcg(&G.state[v]).x);
    }
    if constexpr (FIELDS) batch_fields_epilogue(a, G, q, gthreads, gtid);
    group_sync<CS>();
  }
}

// Single plan on the whole GPU: cooperative launch, one CTA per SM (x occupancy), 8 lanes per
// candidate, grid-wide barrier per round.  Used when latency of ONE wavefront matters.
#ifndef MNB_GRID_MINBLOCKS
#define MNB_GRID_MINBLOCKS 1
#endif
// RESUME: as k_cvp<CS, true> (mnb_cvp_replan)
template <bool RESUME = false>
__global__ void __launch_bounds__(512, MNB_GRID_MINBLOCKS) k_cvp_grid(const CvpKernelArgs a) {
  __shared__ GridStage st;          // + a.slots x GRID_SLOT_BYTES of dynamic shared memory
  uint32_t g, gthreads, gtid;
  group_coords<0>(g, gthreads, gtid);
  GroupCtl* ctl = a.ws.ctl;
  if (threadIdx.x == 0) { stage_init(st); st.dn[0] = 0; st.dn[1] = 0; st.cap = a.slots; }
  __syncthreads();
  CvpEllProblem prob;
  uint32_t rv[3];
  cvp_single_setup<0, RESUME>(a, true, true, gthreads, gtid, prob, rv);
  const float delta = a.delta;      // not clamped to goal_dist_offset: the engine caps settling instead (settle_cap)
  // in-round sweeps pay off once the band is several dependency hops deep.  On the 5 M terrain with 2048 GridStage slots
  // and a 40 w band (29 hops; H100 80GB HBM3, 700 W): 12 / 18 / 24 / 32 / 48 sweeps took 39.3 / 35.7 / 34.6 / 34.9 / 36.2 ms
  // (rounds 189 / 135 / 117 / 112 / 106), so at most 24
  int sweeps = a.sweeps;
  if (sweeps < 0) sweeps = delta < 2.8f * a.hop ? 0 : min(24, (int)(delta / a.hop));
  const float band_init = RESUME ? __uint_as_float(__ldcg(&ctl->lo[2])) : prob.seed_max_d;    // (see k_cvp)
  run_band_rounds_sub8<0, true, CvpEllProblem, RESUME>(prob, ctl, a.ws.list0, a.ws.list1, a.ws.mark, st, delta, gthreads, gtid, a.robot_face >= 0,
                          rv[0], rv[1], rv[2], a.goal_dist_offset, a.cancel_flag, nextafterf(band_init, __uint_as_float(INF_BITS)), a.max_rounds,
                          sweeps, a.V);
  group_sync<0>(ctl->barrier);
  if (a.out_dist)
    for (uint32_t v = gtid; v < a.V; v += gthreads) a.out_dist[v] = __uint_as_float(a.ws.state[v].x);
}

// The epilogue of a single plan (cvp_epilogue_problem above), one thread per vertex; the goal cutoff is the plan's.  In two
// launches: k_cvp_epilogue replays every vertex its ELL row covers, in registers, and lists the others (ws.list1, free once
// the wave has ended; ctl->epi_csr entries, cleared by the host before the launch); k_cvp_epilogue_csr replays those on
// their CSR records.  A call to the out-of-line replay would cost the first kernel its registers: the call convention
// caps them and saves the live ones to a stack frame.  ALL_CSR (mnb_debug_set_cvp_epilogue(ctx, 1), tests only): every
// vertex the row replay covers is listed as well, so that the second launch replays them all on their CSR records.
#ifndef MNB_EPILOGUE_THREADS
#define MNB_EPILOGUE_THREADS 256
#endif
template <bool ALL_CSR = false>
__global__ void __launch_bounds__(MNB_EPILOGUE_THREADS) k_cvp_epilogue(const CvpKernelArgs a, GroupCtl* ctl) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.V) return;
  const uint32_t sf = a.seed_faces[0];
  CvpProblem prob;
  cvp_epilogue_problem(a, a.ws.state, a.ws.ext, a.ws.root, a.ws.chg, a.ws.pool, ctl, sf, a.seed_pos, time_get(ctl->goal_time),
                       a.out_pred, a.out_dir, a.out_cut, prob);
  cvp_epilogue_vertex<true, ALL_CSR>(prob, a.ell_idx, a.ell_w, ctl, sf, __uint_as_float(ctl->goal_bits), c,
                      [&](uint32_t v) { a.ws.list1[atomicAdd(&ctl->epi_csr, 1u)] = v; });
}
__global__ void __launch_bounds__(256) k_cvp_epilogue_csr(const CvpKernelArgs a, GroupCtl* ctl) {
  const uint32_t n = __ldcg(&ctl->epi_csr);
  const uint32_t sf = a.seed_faces[0];
  CvpProblem prob;
  cvp_epilogue_problem(a, a.ws.state, a.ws.ext, a.ws.root, a.ws.chg, a.ws.pool, ctl, sf, a.seed_pos, time_get(ctl->goal_time),
                       a.out_pred, a.out_dir, a.out_cut, prob);
  const float goal = __uint_as_float(ctl->goal_bits);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) prob.epilogue_csr(__ldcg(&a.ws.list1[i]), goal);
}

// ============================================================================
// CVP replan (mnb_cvp_replan): the resident single-plan wave resumes from the earliest pop time a cost change can reach
// (DESIGN §4, "Replan").  Every event of the reference loop before
//   T0 = min(pop times of the closed 1-rings of the changed vertices, the old wave's cutoff arming time,
//            the latest old pop time of the new robot face's vertices)
// reads only labels, gates and weights that did not change, so the vertices that popped before T0 keep their labels and
// the rest of the wave is run again: k_replan_t0 + k_replan_t0_final reduce T0, k_replan_rollback keeps the prefix and
// resets everything else, k_replan_frontier lists the first candidates, and k_cvp_grid<true> / k_cvp<CS, true> resume.
// ============================================================================
struct ReplanArgs {
  uint32_t V;
  const uint32_t* faces; const uint32_t* cor_ptr; const int4* cor_idx;
  const float* cost; const uint8_t* invalid; double cost_limit;
  WaveWorkspace ws;                 // the resident wave (one group)
  const uint32_t* changed; uint32_t n_changed;   // device, any order, duplicates allowed
  uint32_t seed_face;
  long long robot_face;             // -1 = none
  uint32_t* t0;                     // [8 + 6 * blocks of k_replan_t0]: T0, the resume flag, one spare word, the block minima
};
constexpr uint32_t REPLAN_T0_WORDS = 8;

__device__ __forceinline__ LabelStore replan_store(const ReplanArgs& a) {
  LabelStore s;
  s.state = a.ws.state; s.root_arr = a.ws.root; s.ext_arr = a.ws.ext; s.chg = a.ws.chg;
  s.pool = a.ws.pool; s.pool_w = a.ws.pool; s.pool_cap = a.ws.pool_cap; s.pool_top = &a.ws.ctl->pool_top; s.pool_overflow = &a.ws.ctl->pool_overflow;
  return s;
}

// the earliest of the block's times t (every thread calls this; the result is valid in thread 0)
__device__ __forceinline__ EvTime time_min_block(const TimeAlg& A, EvTime t) {
  __shared__ uint32_t sw[32][6];
  for (int o = 16; o > 0; o >>= 1) {
    EvTime u;
    u.a1 = __shfl_down_sync(0xffffffffu, t.a1, o); u.root = __shfl_down_sync(0xffffffffu, t.root, o);
    u.a2 = __shfl_down_sync(0xffffffffu, t.a2, o); u.a3 = __shfl_down_sync(0xffffffffu, t.a3, o);
    u.ext = __shfl_down_sync(0xffffffffu, t.ext, o); u.self = __shfl_down_sync(0xffffffffu, t.self, o);
    if (A.tless(u, t)) t = u;
  }
  if ((threadIdx.x & 31) == 0) time_put(sw[threadIdx.x >> 5], t);
  __syncthreads();
  if (threadIdx.x == 0)
    for (uint32_t w = 1; w < (blockDim.x + 31) / 32; ++w) {
      EvTime u;                          // (plain loads: time_get reads global memory through the L2 only)
      u.a1 = __uint_as_float(sw[w][0]); u.root = sw[w][1]; u.a2 = __uint_as_float(sw[w][2]); u.a3 = __uint_as_float(sw[w][3]);
      u.ext = sw[w][4]; u.self = sw[w][5];
      if (A.tless(u, t)) t = u;
    }
  return t;
}

// The bodies the single replan (k_replan_*) and the batch replan (k_batch_replan_t0, k_cvp_batch_replan) share.
// The earliest finite pop time of S over the changed vertices changed[i0], changed[i0 + stride], ... and their face
// neighbours (time_never() if there is none).
__device__ __forceinline__ EvTime replan_changed_min(const LabelStore& S, const uint32_t* changed, uint32_t n_changed, const uint32_t* cor_ptr,
                                                     const int4* cor_idx, uint32_t i0, uint32_t stride) {
  EvTime best = time_never();
  auto consider = [&](uint32_t x) {
    const Label L = S.load_label(x);
    if (__float_as_uint(L.d) != INF_BITS && S.tless(L.t, best)) best = L.t;
  };
  for (uint32_t i = i0; i < n_changed; i += stride) {
    const uint32_t c = __ldg(&changed[i]);
    consider(c);
    for (uint32_t k = __ldg(&cor_ptr[c]), ke = __ldg(&cor_ptr[c + 1]); k < ke; ++k) {
      const int4 ix = __ldg(&cor_idx[k]);
      consider((uint32_t)ix.x); consider((uint32_t)ix.y);
    }
  }
  return best;
}
// Does every vertex of the seed face sv pop before T0?  (Otherwise the wave runs whole.)
__device__ __forceinline__ bool replan_seeds_before(const LabelStore& S, const uint32_t* sv, const EvTime& T0) {
  bool ok = true;
  for (int k = 0; k < 3; ++k) ok = ok && S.tless(S.load_label(__ldg(&sv[k])).t, T0);
  return ok;
}
// The rollback of vertex v: a vertex that popped before T0 (and every seed vertex sv[]) stays settled with its label, pool
// record included; every other one gets the state of a fresh wave.  Vertices that can never be fixed (invalid, cost >=
// cost_limit) hold +inf and are reset with the rest.
__device__ __forceinline__ void replan_rollback_vertex(const LabelStore& S, const uint32_t* sv, const EvTime& T0, uint32_t* mark, uint32_t v) {
  const bool seed = v == __ldg(&sv[0]) || v == __ldg(&sv[1]) || v == __ldg(&sv[2]);
  const Label L = S.load_label(v);
  const bool keep = seed || (__float_as_uint(L.d) != INF_BITS && S.tless(L.t, T0));
  if (keep) mark[v] = MARK_FIXED;
  else { S.state[v] = state_inf(); mark[v] = MARK_NONE; }
  S.chg[v] = 0u;
}
// The frontier test of vertex v after the rollback (every mark written, a barrier between): a vertex that may take a label
// (as the wave's activation) and shares a face with a kept vertex is a first candidate -- in a fresh wave the kept labels
// would have pulled it in.  It is appended to list0, counted in *count0.
__device__ __forceinline__ void replan_frontier_vertex(const LabelStore& S, const uint32_t* sv, const uint32_t* cor_ptr, const int4* cor_idx,
                                                       const float* cost, const uint8_t* invalid, double cost_limit, uint32_t* mark,
                                                       uint32_t* list0, unsigned int* count0, uint32_t v) {
  const uint32_t mv = __ldcg(&mark[v]);
#ifdef MNB_EMU_ACTIVE
  // the interpreter checks two invariants of the rollback: the seeds stay fixed, and a kept label's level stack names
  // only kept vertices (levels are running maxima of the pop sequence, so they popped before; LabelStore::names relies on it)
  if ((v == sv[0] || v == sv[1] || v == sv[2]) && mv != MARK_FIXED) { fprintf(stderr, "[replan] seed %u not fixed\n", v); abort(); }
  if (mv == MARK_FIXED) {
    const Label L = S.load_label(v);
    for (uint32_t i = 1, n = S.levels_of(L.t); i <= n; ++i) {
      uint32_t kb, id; S.level_of(L.t, i, kb, id);
      if (id != v && mark[id] != MARK_FIXED) { fprintf(stderr, "[replan] kept label of %u names reset vertex %u\n", v, id); abort(); }
    }
  }
#else
  (void)S; (void)sv;
#endif
  if (mv != MARK_NONE) return;
  if (!CvpProblem::eligible(v, cost, invalid, cost_limit)) return;
  bool next_to_kept = false;
  for (uint32_t k = __ldg(&cor_ptr[v]), ke = __ldg(&cor_ptr[v + 1]); k < ke && !next_to_kept; ++k) {
    const int4 ix = __ldg(&cor_idx[k]);
    next_to_kept = __ldcg(&mark[ix.x]) == MARK_FIXED || __ldcg(&mark[ix.y]) == MARK_FIXED;
  }
  if (next_to_kept) {
    mark[v] = MARK_CAND;
    list0[atomicAdd(count0, 1u)] = v;
  }
}

// 1. per block: the earliest pop time over the changed vertices and their face neighbours (labels of the resident wave)
__global__ void __launch_bounds__(256) k_replan_t0(const ReplanArgs a) {
  const LabelStore S = replan_store(a);
  EvTime best = replan_changed_min(S, a.changed, a.n_changed, a.cor_ptr, a.cor_idx, blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x);
  best = time_min_block(S, best);
  if (threadIdx.x == 0) time_put(a.t0 + REPLAN_T0_WORDS + 6 * blockIdx.x, best);
}

// 2. one block: T0 = min(block minima, the old cutoff's arming time, the new cutoff's arming time if the old wave knows
//    it); t0[6] = 1 if every seed pops before T0 (otherwise the call runs a whole wave)
__global__ void __launch_bounds__(256) k_replan_t0_final(const ReplanArgs a, uint32_t blocks) {
  const LabelStore S = replan_store(a);
  EvTime best = time_never();
  for (uint32_t b = threadIdx.x; b < blocks; b += blockDim.x) {
    const EvTime u = time_get(a.t0 + REPLAN_T0_WORDS + 6 * b);
    if (S.tless(u, best)) best = u;
  }
  best = time_min_block(S, best);
  if (threadIdx.x != 0) return;
  // the old wave's goal cutoff: events after its arming differ with another robot face or offset (+inf key: not armed)
  const EvTime armed = time_get(a.ws.ctl->goal_time);
  if (__float_as_uint(armed.a1) != INF_BITS && S.tless(armed, best)) best = armed;
  // the new goal cutoff arms when the last vertex of the robot face pops: if all three popped in the old wave before
  // T0, that moment is the same in a fresh wave, and the events after it differ
  if (a.robot_face >= 0) {
    EvTime late = ev_normal(0.0f, 0u); bool all = true;
    for (int k = 0; k < 3; ++k) {
      const Label L = S.load_label(__ldg(&a.faces[3 * (size_t)a.robot_face + k]));
      if (__float_as_uint(L.d) == INF_BITS) all = false;
      else if (k == 0 || S.tless(late, L.t)) late = L.t;
    }
    if (all && S.tless(late, best)) best = late;
  }
  const bool ok = replan_seeds_before(S, a.faces + 3 * (size_t)a.seed_face, best);
  time_put(a.t0, best);
  a.t0[6] = ok ? 1u : 0u;
}

// 3. the rollback (replan_rollback_vertex).  The group's control block is reset for the round loop with the band at T0;
//    the level pool keeps its records and allocation continues from its top.
__global__ void __launch_bounds__(256) k_replan_rollback(const ReplanArgs a) {
  const LabelStore S = replan_store(a);
  const EvTime T0 = time_get(a.t0);
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v == 0) {
    GroupCtl* ctl = a.ws.ctl;
    const unsigned int top = ctl->pool_top;
    *ctl = GroupCtl{};
    ctl_reset(ctl, 0u, T0.a1);
    ctl->pool_top = top;
  }
  if (v >= a.V) return;
  replan_rollback_vertex(S, a.faces + 3 * (size_t)a.seed_face, T0, a.ws.mark, v);
  a.ws.ver[v] = 0u;
}

// 4. the first candidates (replan_frontier_vertex)
__global__ void __launch_bounds__(256) k_replan_frontier(const ReplanArgs a) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.V) return;
  replan_frontier_vertex(replan_store(a), a.faces + 3 * (size_t)a.seed_face, a.cor_ptr, a.cor_idx, a.cost, a.invalid, a.cost_limit, a.ws.mark,
                         a.ws.list0, &a.ws.ctl->count[0], v);
}

// ============================================================================
// Batch replan (mnb_cvp_batch_replan): full-field waves of many goals resume from their own T0 (DESIGN §4, "Batch
// replan").  Without a goal cutoff, T0 is the earliest old pop time in the closed 1-rings of the changed vertices.  The
// resident waves live in slots, one device allocation each; the host uploads one BatchReplanGoal per distinct goal.
// ============================================================================
// One resident slot: the wave's labels and side arrays, its pred / dir / cut rows and its level pool, then a 16-byte
// header (the pool top after the wave) -- 36 bytes per vertex, the pool's 4 * pool_cap bytes and the header.
struct ReplanSlot {
  uint4* state; uint32_t* ext; uint32_t* root; uint32_t* pred; float* dir; int32_t* cut; uint32_t* pool; uint32_t* pool_top;
};
__host__ __device__ __forceinline__ size_t replan_slot_bytes(uint32_t V, uint32_t pool_cap) {
  return (size_t)V * (sizeof(uint4) + 5 * sizeof(uint32_t)) + (size_t)pool_cap * sizeof(uint32_t) + 16;
}
__device__ __forceinline__ ReplanSlot replan_slot(uint8_t* base, uint32_t V, uint32_t pool_cap) {
  ReplanSlot s;
  s.state = reinterpret_cast<uint4*>(base);
  uint32_t* w = reinterpret_cast<uint32_t*>(base + (size_t)V * sizeof(uint4));
  s.ext = w; s.root = w + V; s.pred = w + 2 * (size_t)V; s.dir = reinterpret_cast<float*>(w + 3 * (size_t)V);
  s.cut = reinterpret_cast<int32_t*>(w + 4 * (size_t)V); s.pool = w + 5 * (size_t)V; s.pool_top = s.pool + pool_cap;
  return s;
}

// one distinct goal of a call (q: its index in the call's seed arrays), built by the host
struct BatchReplanGoal {
  uint8_t* slot;                // its resident slot, or null: the wave runs whole in the workspace
  uint32_t row;                 // the caller's row it writes (the host copies it to the rows of duplicate goals)
  uint32_t resume;              // 1 when uploaded: the slot holds this goal's wave of the same costs and cost limit.
                                // k_batch_replan_t0 leaves it at 1 only if the wave can resume.
  uint32_t t0[6];               // T0 (k_batch_replan_t0)
  unsigned int chunks_done;     // k_batch_replan_t0's finished blocks of this goal (0 when uploaded)
};

struct BatchReplanT0Args {
  uint32_t V, pool_cap;
  const uint32_t* faces; const uint32_t* cor_ptr; const int4* cor_idx;
  BatchReplanGoal* goals; const uint32_t* seed_faces;
  const uint32_t* changed; uint32_t n_changed;   // device, any order, duplicates allowed
  uint32_t chunks;              // blocks per goal: block b serves goal b / chunks
  uint32_t* minima;             // [goals][chunks] pop times (6 words)
};

// the label store of a batch wave's labels (chg and the pool top: the group's; k_batch_replan_t0 only reads the labels)
__device__ __forceinline__ LabelStore batch_store(uint4* state, uint32_t* ext, uint32_t* root, uint32_t* pool, uint32_t pool_cap, uint32_t* chg,
                                                  GroupCtl* ctl) {
  LabelStore S;
  S.state = state; S.root_arr = root; S.ext_arr = ext; S.chg = chg; S.pool = pool; S.pool_w = pool; S.pool_cap = pool_cap;
  S.pool_top = ctl ? &ctl->pool_top : nullptr; S.pool_overflow = ctl ? &ctl->pool_overflow : nullptr;
  return S;
}

// T0 of every goal that may resume, in one launch over (goal, chunk of the changed list): each block reduces its chunk;
// the last block of a goal reduces the chunk minima and sets the resume flag -- every seed pops before T0 and the slot's
// level pool is at most half full.  No changed vertex: T0 is "never", and the resumed wave re-runs nothing.
__global__ void __launch_bounds__(256) k_batch_replan_t0(const BatchReplanT0Args a) {
  const uint32_t q = blockIdx.x / a.chunks, chunk = blockIdx.x % a.chunks;
  BatchReplanGoal* gq = a.goals + q;
  if (!gq->resume) return;                                       // (block-uniform: a host value)
  const ReplanSlot sl = replan_slot(gq->slot, a.V, a.pool_cap);
  const LabelStore S = batch_store(sl.state, sl.ext, sl.root, sl.pool, a.pool_cap, nullptr, nullptr);
  EvTime best = replan_changed_min(S, a.changed, a.n_changed, a.cor_ptr, a.cor_idx, chunk * blockDim.x + threadIdx.x, a.chunks * blockDim.x);
  best = time_min_block(S, best);
  __shared__ bool last;
  if (threadIdx.x == 0) {
    time_put(a.minima + 6 * (size_t)blockIdx.x, best);
    __threadfence();                                             // the minimum before the count that publishes it
    last = atomicAdd(&gq->chunks_done, 1u) == a.chunks - 1;
  }
  __syncthreads();
  if (threadIdx.x != 0 || !last) return;
  __threadfence();
  for (uint32_t b = 0; b < a.chunks; ++b) {
    const EvTime u = time_get(a.minima + 6 * ((size_t)q * a.chunks + b));
    if (S.tless(u, best)) best = u;
  }
  time_put(gq->t0, best);
  const bool room = __ldcg(sl.pool_top) <= a.pool_cap / 2;
  gq->resume = room && replan_seeds_before(S, a.faces + 3 * (size_t)a.seed_faces[q], best) ? 1u : 0u;
}

struct CvpBatchReplanArgs : CvpKernelArgs {
  const BatchReplanGoal* goals; // [n_queries]
  uint32_t pool_room;           // level-pool words a resumed wave may add (mnb_debug_set_replan_pool_room; 0 = the pool's)
};

// The rollback and the frontier of a resumed goal (seed face sv) on the group's labels G (a slot), then the control block
// for the round loop with the band at T0 and the slot's pool top.  Called by every thread of the group; ends with a group
// barrier.  Out of line, as the batch kernel's other once-per-wave work.
template <int CS>
__device__ __noinline__ void batch_replan_rollback(const CvpBatchReplanArgs& a, const BatchGroup& G, uint32_t* list0, const uint32_t* sv,
                                                   const EvTime& T0, const uint32_t* pool_top, uint32_t gthreads, uint32_t gtid) {
  const LabelStore S = batch_store(G.state, G.ext_arr, G.root_arr, G.pool, G.pool_cap, G.chg, G.ctl);
  for (uint32_t v = gtid; v < a.V; v += gthreads) {
    replan_rollback_vertex(S, sv, T0, G.mark, v);
    G.skipw[v] = make_uint4(INF_BITS, INF_BITS, 0u, 0u);
  }
  if (gtid == 0) {
    ctl_reset(G.ctl, 0u, T0.a1);
    G.ctl->pool_top = __ldcg(pool_top);
  }
  group_sync<CS>();
  for (uint32_t v = gtid; v < a.V; v += gthreads)
    replan_frontier_vertex(S, sv, a.cor_ptr, a.cor_idx, a.cost, a.invalid, a.cost_limit, G.mark, list0, &G.ctl->count[0], v);
  group_sync<CS>();
}

// The clearing pass and the seeding of a whole wave for goal q (as k_cvp_batch's); retry: the goal's resumed wave
// overflowed the level pool, and the flag is cleared (after the barrier of the clearing pass: every thread of the group
// has read it).  Called by every thread of the group; ends with a group barrier.
template <int CS>
__device__ __noinline__ void batch_replan_seed(const CvpBatchReplanArgs& a, const BatchGroup& G, uint32_t* list0, uint32_t q, bool retry,
                                               uint32_t gthreads, uint32_t gtid) {
  for (uint32_t v = gtid; v < a.V; v += gthreads) { G.state[v] = state_inf(); G.mark[v] = MARK_NONE; G.chg[v] = 0u; G.skipw[v] = make_uint4(INF_BITS, INF_BITS, 0u, 0u); }
  group_sync<CS>();
  if (gtid == 0) {
    if (retry) G.ctl->pool_overflow = 0u;
    const CvpSeeds cs = cvp_seeds(a.faces, a.pos, a.cost, a.invalid, a.cost_limit, a.seed_faces[q], a.seed_pos + 3 * (size_t)q);
    CvpEllProblem prob;
    batch_make_problem(a, G, cs, 0, prob);
    seed_wave(prob, G.ctl, G.mark, list0, cs.s, cs.d, 3, cs.seed_min);
  }
  group_sync<CS>();
}

// The epilogue of goal q into pred / dir / cut (any may be null).  TAIL (a resumed wave): the kept vertices (MARK_FIXED)
// are skipped -- they popped before T0, so none of their faces changed and their sources popped before them: their
// entries in the slot's rows are still exact.
__device__ __noinline__ void batch_replan_epilogue(const CvpKernelArgs& a, const BatchGroup& G, uint32_t q, uint32_t* pred, float* dir, int32_t* cut,
                                                   bool tail, uint32_t gthreads, uint32_t gtid) {
  const uint32_t sf = a.seed_faces[q];
  CvpProblem prob;
  cvp_epilogue_problem(a, G.state, G.ext_arr, G.root_arr, G.chg, G.pool, G.ctl, sf, a.seed_pos + 3 * (size_t)q, ev_normal(__uint_as_float(INF_BITS), 0u),
                       pred, dir, cut, prob);
  for (uint32_t v = gtid; v < a.V; v += gthreads)
    if (!(tail && __ldcg(&G.mark[v]) == MARK_FIXED))
      cvp_epilogue_vertex<false>(prob, a.ell_idx, a.ell_w, G.ctl, sf, __uint_as_float(INF_BITS), v, [](uint32_t) {});
}

// The batch replan: k_cvp_batch<CS, true> over the distinct goals of a.goals.  A goal with a slot keeps its labels, side
// arrays, level pool and rows there; marks, chg, skipw and the lists are the group's workspace, as for a goal without
// one.  A goal whose flag k_batch_replan_t0 left raised resumes from T0: rollback and frontier, the round loop with the band
// just above T0 (stopping if the level pool overflows; then the goal runs again as a whole wave from an empty pool), and
// the epilogue of the re-run tail alone.  Every other goal runs a whole wave.  No goal is taken once the cancel flag is set.
template <int CS>
__global__ void __launch_bounds__(MNB_BATCH_THREADS, MNB_BATCH_MINBLOCKS) k_cvp_batch_replan(const CvpBatchReplanArgs a) {
  __shared__ BatchStage st;
  __shared__ BatchWork wk;
  uint32_t g, gthreads, gtid;
  group_coords<CS>(g, gthreads, gtid);
  const uint32_t V = a.V;
  BatchGroup W;
  W.state = a.ws.state + (size_t)g * V; W.root_arr = a.ws.root + (size_t)g * V; W.ext_arr = a.ws.ext + (size_t)g * V;
  W.chg = a.ws.chg + (size_t)g * V; W.mark = a.ws.mark + (size_t)g * V; W.pool = a.ws.pool + (size_t)g * a.ws.pool_cap;
  W.pool_cap = a.ws.pool_cap; W.ctl = a.ws.ctl + g; W.skipw = a.ws.skipw + (size_t)g * V;
  uint32_t* list0 = a.ws.list0 + (size_t)g * V;
  uint32_t* list1 = a.ws.list1 + (size_t)g * V;
  GroupCtl* ctl = W.ctl;
  if (threadIdx.x == 0) { stage_init(st); wk.n = 0; wk.ns = 0; }
  __syncthreads();
  for (;;) {
    if (gtid == 0) ctl->query = (a.cancel_flag && *(const volatile int*)a.cancel_flag) ? a.n_queries : atomicAdd(a.next_query, 1u);
    group_sync<CS>();
    const uint32_t q = __ldcg(&ctl->query);
    if (q >= a.n_queries) break;
    const BatchReplanGoal* gq = a.goals + q;
    uint8_t* const slot_base = gq->slot;
    BatchGroup G = W;
    ReplanSlot sl{};
    if (slot_base) {
      sl = replan_slot(slot_base, V, a.ws.pool_cap);
      G.state = sl.state; G.ext_arr = sl.ext; G.root_arr = sl.root; G.pool = sl.pool;
    }
    const SeedFace sd = cvp_seeds(a.faces, a.pos, a.cost, a.invalid, a.cost_limit, a.seed_faces[q], a.seed_pos + 3 * (size_t)q);
    // (a pool overflow of an earlier goal of the group fails the call: its goals then run whole, and nothing is retried)
    bool resume = slot_base && gq->resume && !__ldcg(&ctl->pool_overflow), retry = false;
    for (;;) {
      float band_init;
      if (resume) {
        const EvTime T0 = time_get(gq->t0);
        batch_replan_rollback<CS>(a, G, list0, a.faces + 3 * (size_t)a.seed_faces[q], T0, sl.pool_top, gthreads, gtid);
        if (a.pool_room) G.pool_cap = min(G.pool_cap, __ldcg(&ctl->pool_top) + a.pool_room);
        band_init = T0.a1;
      } else {
        batch_replan_seed<CS>(a, G, list0, q, retry, gthreads, gtid);
        band_init = sd.seed_max;
      }
      run_band_rounds_batch<CS, false, true>(a, G, list0, list1, st, wk, a.delta, gthreads, gtid, sd, nextafterf(band_init, __uint_as_float(INF_BITS)));
      group_sync<CS>();
      if (!resume || !__ldcg(&ctl->pool_overflow)) break;
      // the resumed wave ran out of level pool: the goal runs again as a whole wave from an empty pool (seed_wave resets
      // the pool top)
      resume = false; retry = true;
      G.pool_cap = a.ws.pool_cap;
    }
    const size_t row = (size_t)gq->row * V;
    uint32_t* const o_pred = a.out_pred ? a.out_pred + row : nullptr;
    float* const o_dir = a.out_dir ? a.out_dir + row : nullptr;
    int32_t* const o_cut = a.out_cut ? a.out_cut + row : nullptr;
    if (slot_base) {
      // the slot's rows are completed (the re-run tail, or every vertex), then copied to the caller's
      batch_replan_epilogue(a, G, q, sl.pred, sl.dir, sl.cut, resume, gthreads, gtid);
      group_sync<CS>();
      for (uint32_t v = gtid; v < V; v += gthreads) {
        if (o_pred) o_pred[v] = __ldcg(&sl.pred[v]);
        if (o_dir) o_dir[v] = __ldcg(&sl.dir[v]);
        if (o_cut) o_cut[v] = __ldcg(&sl.cut[v]);
      }
      if (gtid == 0) *sl.pool_top = ctl->pool_top;
    } else if (o_pred || o_dir || o_cut) {
      batch_replan_epilogue(a, G, q, o_pred, o_dir, o_cut, false, gthreads, gtid);
    }
    if (a.out_dist) {
      float* od = a.out_dist + row;
      for (uint32_t v = gtid; v < V; v += gthreads) od[v] = __uint_as_float(__ldcg(&G.state[v]).x);
    }
    group_sync<CS>();
  }
}

// start == goal (dijkstra_mesh_planner.cpp:252-255): the maps as the reference leaves them after clearing (:241-249)
__global__ void k_dijkstra_trivial(uint32_t V, uint32_t seed, float* __restrict__ dist, uint32_t* __restrict__ pred) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  if (dist) dist[v] = v == seed ? 0.0f : __uint_as_float(INF_BITS);
  if (pred) pred[v] = v;
}

struct DijkstraKernelArgs {
  uint32_t V;
  const uint32_t* adj_ptr; const uint2* adj_nw;
  const float* cost; const uint8_t* invalid;
  WaveWorkspace ws;
  uint32_t seed_vertex; long long robot_vertex;
  double cost_limit, goal_dist_offset;
  float delta;
  float* out_dist; uint32_t* out_pred;
  const int* cancel_flag;
  uint32_t max_rounds;
  const uint4* ell_adj; int sweeps; float hop; uint32_t slots;   // whole-grid kernel only (slots: see k_cvp_grid)
};

// The prologue of a single-plan Dijkstra wave (k_dijkstra, k_dijkstra_grid): the clearing pass (the sweep versions only for
// the kernel with in-round sweeps), the problem, the seed (dijkstra:276, d = 0) with its first candidates, and the robot
// vertex still to settle.  Called by every thread of the group; ends with a group barrier.
template <int CS>
__device__ __forceinline__ void dijkstra_single_setup(const DijkstraKernelArgs& a, bool clear_ver, uint32_t gthreads, uint32_t gtid,
                                                      DijkstraProblem& prob) {
  for (uint32_t v = gtid; v < a.V; v += gthreads) {
    a.ws.state[v] = state_inf(); a.ws.mark[v] = MARK_NONE; a.out_pred[v] = v;
    if (clear_ver) a.ws.ver[v] = 0u;
  }
  group_sync<CS>();
  prob.adj_ptr = a.adj_ptr; prob.adj_nw = a.adj_nw; prob.cost = a.cost; prob.invalid = a.invalid;
  prob.state = a.ws.state; prob.pred = a.out_pred; prob.cost_limit = a.cost_limit; prob.deferred_m = __uint_as_float(INF_BITS); prob.strict = 0;
  if (gtid == 0) {
    const float d0 = 0.0f;
    seed_wave(prob, a.ws.ctl, a.ws.mark, a.ws.list0, &a.seed_vertex, &d0, 1, 0.0f);
    if (a.robot_vertex >= 0) a.ws.ctl->robot_left = 1;
  }
  group_sync<CS>();
}

template <int CS>
__global__ void __launch_bounds__(512, 1) k_dijkstra(const DijkstraKernelArgs a) {
  __shared__ Stage st;
  uint32_t g, gthreads, gtid;
  group_coords<CS>(g, gthreads, gtid);
  if (threadIdx.x == 0) stage_init(st);
  __syncthreads();
  DijkstraProblem prob;
  dijkstra_single_setup<CS>(a, false, gthreads, gtid, prob);
  const int has_robot = a.robot_vertex >= 0;
  const uint32_t rv = has_robot ? (uint32_t)a.robot_vertex : 0xffffffffu;
  float delta = a.delta;
  if (has_robot && a.goal_dist_offset < (double)delta) delta = (float)fmax(a.goal_dist_offset, 1e-4);
  run_band_rounds<CS>(prob, a.ws.ctl, a.ws.list0, a.ws.list1, a.ws.mark, st, delta, gthreads, gtid, has_robot, rv, rv, rv,
                      a.goal_dist_offset, a.cancel_flag, 1e-30f, a.max_rounds);
  group_sync<CS>();
  for (uint32_t v = gtid; v < a.V; v += gthreads) a.out_dist[v] = __uint_as_float(a.ws.state[v].x);
}

// Batches of full-field Dijkstra plans (mnb_dijkstra_batch): the outer loop of k_cvp_batch around the round loop of
// k_dijkstra.  One wavefront per CTA (CS = 1) or per cluster of CS CTAs; persistent groups pull seed indices from an
// atomic counter and stop taking new ones once the cancel flag is set.  A wavefront owns only what the round loop reads:
// the float label (tau = d), the marks, two candidate lists and its GroupCtl -- 16 bytes per vertex.  Row q of the
// outputs is written by the group that ran seed q; out_pred (may be null) doubles as the problem's predecessor array.
struct DijkstraBatchWorkspace {   // per group (index g): label + g*V etc.
  float* label;
  uint32_t* mark;
  uint32_t* list0;
  uint32_t* list1;
  GroupCtl* ctl;
};
constexpr size_t DIJKSTRA_BATCH_BYTES_PER_VERTEX = sizeof(float) + 3 * sizeof(uint32_t);

struct DijkstraBatchArgs {
  uint32_t V;
  const uint32_t* adj_ptr; const uint2* adj_nw;
  const float* cost; const uint8_t* invalid;
  DijkstraBatchWorkspace ws;
  uint32_t n_queries;
  const uint32_t* seeds;        // [n_queries] device
  double cost_limit;
  float delta;
  float* out_dist;              // [n_queries][V] or null
  uint32_t* out_pred;           // [n_queries][V] or null
  unsigned int* next_query;
  const int* cancel_flag;
  uint32_t max_rounds;
  TargetSet tg;                 // k_dijkstra_batch<CS, true> only
};

// MATRIX (mnb_dijkstra_matrix): a wave ends once the target vertices of a.tg have settled and writes their distances, row
// q of a.tg.out, instead of the V-sized rows.
template <int CS, bool MATRIX = false>
__global__ void __launch_bounds__(MNB_BATCH_THREADS, MNB_BATCH_MINBLOCKS) k_dijkstra_batch(const DijkstraBatchArgs a) {
  __shared__ Stage st;
  uint32_t g, gthreads, gtid;
  group_coords<CS>(g, gthreads, gtid);
  const uint32_t V = a.V;
  float* label = a.ws.label + (size_t)g * V;
  uint32_t* mark = a.ws.mark + (size_t)g * V;
  uint32_t* list0 = a.ws.list0 + (size_t)g * V;
  uint32_t* list1 = a.ws.list1 + (size_t)g * V;
  GroupCtl* ctl = a.ws.ctl + g;
  const volatile int* cancel = a.cancel_flag;
  if (threadIdx.x == 0) stage_init(st);
  __syncthreads();
  DijkstraProblemT<float> prob;
  prob.adj_ptr = a.adj_ptr; prob.adj_nw = a.adj_nw; prob.cost = a.cost; prob.invalid = a.invalid;
  prob.state = label; prob.cost_limit = a.cost_limit; prob.deferred_m = __uint_as_float(INF_BITS);
  for (;;) {
    if (gtid == 0) ctl->query = (cancel && *cancel) ? a.n_queries : atomicAdd(a.next_query, 1u);
    group_sync<CS>();
    const uint32_t q = __ldcg(&ctl->query);
    if (q >= a.n_queries) break;
    uint32_t* pred = a.out_pred ? a.out_pred + (size_t)q * V : nullptr;
    for (uint32_t v = gtid; v < V; v += gthreads) {
      label[v] = __uint_as_float(INF_BITS); mark[v] = MARK_NONE;
      if (pred) pred[v] = v;                                   // dijkstra:268-269
    }
    group_sync<CS>();
    prob.pred = pred;
    if (gtid == 0) {
      const float d0 = 0.0f;                                   // dijkstra:276
      seed_wave(prob, ctl, mark, list0, &a.seeds[q], &d0, 1, 0.0f);
      if constexpr (MATRIX) ctl->targets_left = (int)a.tg.distinct;
    }
    group_sync<CS>();
    if constexpr (MATRIX) {
      // over-cost vertices are eligible: they get labels and settle like any other
      count_targets_done_at_init(a.tg, ctl, mark, V, gthreads, gtid, [&](uint32_t v) { return prob.eligible(v); });
      group_sync<CS>();
    }
    run_band_rounds<CS, MATRIX>(prob, ctl, list0, list1, mark, st, a.delta, gthreads, gtid, 0, 0xffffffffu, 0xffffffffu, 0xffffffffu,
                                0.0, a.cancel_flag, 1e-30f, a.max_rounds, a.tg.bits);
    group_sync<CS>();
    if constexpr (MATRIX) {
      float* om = a.tg.out + (size_t)q * a.tg.m;
      for (uint32_t j = gtid; j < a.tg.m; j += gthreads) om[j] = __ldcg(&label[a.tg.list[j]]);
    } else if (a.out_dist) {
      float* od = a.out_dist + (size_t)q * V;
      for (uint32_t v = gtid; v < V; v += gthreads) od[v] = __ldcg(&label[v]);
    }
    group_sync<CS>();
  }
}

// Field repair (mnb_dijkstra_batch_repair): row q of out_dist / out_pred holds the field of seeds[q] on the costs before
// an update of the vertices in chg, and is brought up to date in place.
struct RepairSet {
  const uint32_t* list;         // [n] device: the distinct changed vertices
  const uint32_t* bits;         // [V/32 + 1] device: their bitmap
  uint32_t n;
  unsigned int* log_n;          // [groups] device: length of the group's log of marked vertices (zero between waves)
};
struct DijkstraRepairArgs : DijkstraBatchArgs {
  RepairSet chg;
};

// The final field is a function of the weights, the gates and the seed alone, so the repair re-runs the wave from the
// old labels that are still realizable (DESIGN §4):
//  1. D = the changed vertices and their descendants in the old predecessor tree, found level by level (x is a child of u
//     iff pred[x] == u), without the seed.  D gets +inf and pred = self.  Every other label is the float sum of a path
//     whose weights and gates did not change: an upper bound of the new distance.
//  2. The first candidates are the changed vertices, their neighbours and the vertices of D next to a finite label that
//     expands.  They are evaluated once without the band filter, so a candidate whose source lies beyond the band holds a
//     finite label from the start; the band starts at the smallest label of the list.  A candidate that changes pulls its
//     neighbours in, as in the round loop.
//  3. The round loop of the batch (run_band_rounds with DijkstraRepairProblem): labels never rise, and a candidate
//     activates its ring when its label first changes.
//  4. The marks the wave set are reset through its log: the mark array is clean between waves without a V-sized pass.
// The label workspace is not used by the repair (the rows are the labels); its first V words of the group hold the log.
template <int CS>
__global__ void __launch_bounds__(MNB_BATCH_THREADS, MNB_BATCH_MINBLOCKS) k_dijkstra_batch_repair(const DijkstraRepairArgs a) {
  __shared__ Stage st;
  __shared__ float s_lo;
  uint32_t g, gthreads, gtid;
  group_coords<CS>(g, gthreads, gtid);
  const uint32_t V = a.V;
  uint32_t* mark = a.ws.mark + (size_t)g * V;
  uint32_t* list0 = a.ws.list0 + (size_t)g * V;
  uint32_t* list1 = a.ws.list1 + (size_t)g * V;
  GroupCtl* ctl = a.ws.ctl + g;
  const volatile int* cancel = a.cancel_flag;
  if (threadIdx.x == 0) stage_init(st);
  __syncthreads();
  DijkstraRepairProblem prob;
  prob.adj_ptr = a.adj_ptr; prob.adj_nw = a.adj_nw; prob.cost = a.cost; prob.invalid = a.invalid;
  prob.cost_limit = a.cost_limit; prob.deferred_m = __uint_as_float(INF_BITS);
  prob.log = reinterpret_cast<uint32_t*>(a.ws.label) + (size_t)g * V; prob.log_n = a.chg.log_n + g;
  const float INF = __uint_as_float(INF_BITS);
  auto changed_vertex = [&](uint32_t x) { return (__ldg(&a.chg.bits[x >> 5]) >> (x & 31)) & 1u; };
  auto expands = [&](uint32_t u) { return (double)__ldg(&a.cost[u]) <= a.cost_limit; };
  for (;;) {
    if (gtid == 0) ctl->query = (cancel && *cancel) ? a.n_queries : atomicAdd(a.next_query, 1u);
    group_sync<CS>();
    const uint32_t q = __ldcg(&ctl->query);
    if (q >= a.n_queries) break;
    float* dist = a.out_dist + (size_t)q * V;
    uint32_t* pred = a.out_pred + (size_t)q * V;
    prob.state = dist; prob.pred = pred;
    const uint32_t s = a.seeds[q];
    // Before the round loop the rings of the GroupCtl serve as scratch (ctl_reset sets them for the loop): lo[] counts
    // the levels of D, count[0] the candidates, m_tau[1] holds their smallest label.
    // 1. D, breadth-first in list1: level 0 the changed vertices (the seed among them only to find its children).  The
    //    children of level k are counted in lo[k % 3]; thread 0 clears the slot of level k + 1 while level k runs, when
    //    the last reads of that slot (level k - 2) are behind a barrier.
    for (uint32_t i = gtid; i < a.chg.n; i += gthreads) list1[i] = a.chg.list[i];
    if (gtid == 0) { ctl->lo[0] = 0u; ctl->count[0] = 0u; ctl->m_tau[1] = INF_BITS; mark[s] = MARK_FIXED; }
    group_sync<CS>();
    uint32_t lb = 0, le = a.chg.n;
    for (uint32_t lvl = 0; lb < le; ++lvl) {
      unsigned int* cnt = &ctl->lo[lvl % 3];
      if (gtid == 0) ctl->lo[(lvl + 1) % 3] = 0u;
      for (uint32_t i = lb + gtid; i < le; i += gthreads) {
        const uint32_t u = __ldcg(&list1[i]);
        prob.activate(u, [&](uint32_t x) {
          if (__ldcg(&pred[x]) == u && !changed_vertex(x)) list1[le + atomicAdd(cnt, 1u)] = x;
        });
      }
      group_sync<CS>();
      lb = le; le += __ldcg(cnt);
    }
    const uint32_t nd = le;
    for (uint32_t i = gtid; i < nd; i += gthreads) {
      const uint32_t x = __ldcg(&list1[i]);
      if (x != s) { dist[x] = INF; pred[x] = x; }
    }
    group_sync<CS>();
    // 2. the first candidates in list0 (marked and logged), then one evaluation without the band filter
    auto add = [&](uint32_t x) {
      if (x != s && __ldcg(&mark[x]) == MARK_NONE && prob.eligible(x) && atomicCAS(&mark[x], MARK_NONE, MARK_CAND) == MARK_NONE) {
        prob.log_mark(x);
        list0[atomicAdd(&ctl->count[0], 1u)] = x;
      }
    };
    for (uint32_t i = gtid; i < a.chg.n; i += gthreads) {
      const uint32_t c = a.chg.list[i];
      add(c);
      prob.activate(c, add);
    }
    for (uint32_t i = gtid; i < nd; i += gthreads) {
      const uint32_t x = __ldcg(&list1[i]);
      bool next_to_source = false;
      prob.activate(x, [&](uint32_t u) { next_to_source |= __float_as_uint(__ldcg(&dist[u])) != INF_BITS && expands(u); });
      if (next_to_source) add(x);
    }
    group_sync<CS>();
    const uint32_t n_first = __ldcg(&ctl->count[0]);
    unsigned long long evals = 0;
    for (uint32_t i = gtid; i < n_first; i += gthreads) {
      const uint32_t c = __ldcg(&list0[i]);
      float nv, ntau;
      evals++;
      if (prob.recompute(c, INF, INF, 0, prob.load_label(c), nv, ntau)) {
        mark[c] = MARK_CAND_ACT;
        prob.activate(c, add);
      }
    }
    if (evals) atomicAdd(&ctl->recomputes, evals);
    if (threadIdx.x == 0) s_lo = INF;
    group_sync<CS>();
    const uint32_t n0 = __ldcg(&ctl->count[0]);
    float my_lo = INF;
    for (uint32_t i = gtid; i < n0; i += gthreads) my_lo = fminf(my_lo, __ldcg(&dist[__ldcg(&list0[i])]));
    const unsigned int wl = __reduce_min_sync(0xffffffffu, __float_as_uint(my_lo));
    if ((threadIdx.x & 31) == 0 && wl != INF_BITS) atomicMin(reinterpret_cast<unsigned int*>(&s_lo), wl);
    __syncthreads();
    if (threadIdx.x == 0 && __float_as_uint(s_lo) != INF_BITS) atomicMin(&ctl->m_tau[1], __float_as_uint(s_lo));
    group_sync<CS>();
    // 3. the round loop from the smallest label of the list (ctl->m_tau[1] served as the group's minimum)
    if (gtid == 0) {
      const float lo0 = __uint_as_float(__ldcg(&ctl->m_tau[1]));
      ctl_reset(ctl, n0, lo0);
    }
    group_sync<CS>();
    run_band_rounds<CS>(prob, ctl, list0, list1, mark, st, a.delta, gthreads, gtid, 0, 0xffffffffu, 0xffffffffu, 0xffffffffu,
                        0.0, a.cancel_flag, 1e-30f, a.max_rounds);
    group_sync<CS>();
    // 4. the marks back to MARK_NONE for the next wave
    const uint32_t nl = __ldcg(prob.log_n);
    for (uint32_t i = gtid; i < nl; i += gthreads) mark[__ldcg(&prob.log[i])] = MARK_NONE;
    if (gtid == 0) mark[s] = MARK_NONE;
    group_sync<CS>();
    if (gtid == 0) *prob.log_n = 0u;
  }
}

// Single Dijkstra plan on the whole GPU: 8 lanes per candidate (one edge each), wide band + in-round sweeps,
// same engine instance as k_cvp_grid.
__global__ void __launch_bounds__(512, 1) k_dijkstra_grid(const DijkstraKernelArgs a) {
  __shared__ GridStage st;          // + a.slots x GRID_SLOT_BYTES of dynamic shared memory
  uint32_t g, gthreads, gtid;
  group_coords<0>(g, gthreads, gtid);
  if (threadIdx.x == 0) { stage_init(st); st.dn[0] = 0; st.dn[1] = 0; st.cap = a.slots; }
  __syncthreads();
  DijkstraEllProblem prob;
  dijkstra_single_setup<0>(a, true, gthreads, gtid, prob);
  prob.ell_adj = a.ell_adj; prob.ver = a.ws.ver;
  const int has_robot = a.robot_vertex >= 0;
  const uint32_t rv = has_robot ? (uint32_t)a.robot_vertex : 0xffffffffu;
  const float delta = a.delta;      // not clamped to goal_dist_offset: the engine caps settling instead (settle_cap)
  int sweeps = a.sweeps;
  // (at most 15: with 2048 slots and a 40 w band on the 5 M terrain 15 / 24 / 36 sweeps took 11.1 / 11.7 / 12.9 ms)
  if (sweeps < 0) sweeps = delta < 2.8f * a.hop ? 0 : min(15, (int)(delta / a.hop));
  run_band_rounds_sub8<0, true>(prob, a.ws.ctl, a.ws.list0, a.ws.list1, a.ws.mark, st, delta, gthreads, gtid, has_robot, rv, rv, rv,
                                a.goal_dist_offset, a.cancel_flag, 1e-30f, a.max_rounds, sweeps, a.V);
  group_sync<0>(a.ws.ctl->barrier);
  for (uint32_t v = gtid; v < a.V; v += gthreads) a.out_dist[v] = __uint_as_float(a.ws.state[v].x);
}
