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
  ctl->goal_time[0] = INF_BITS; ctl->goal_time[1] = 0u; ctl->goal_time[2] = 0u; ctl->goal_time[3] = 0u; ctl->goal_time[4] = 0u; ctl->goal_time[5] = 0u;
  ctl->pool_top = 0u;
  ctl->done_ring[0] = 0u; ctl->done_ring[1] = 0u;
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
template <int CS>
__global__ void __launch_bounds__(MNB_CVP_THREADS, MNB_CVP_MINBLOCKS) k_cvp(const CvpKernelArgs a) {
  __shared__ Stage st;
  uint32_t g, gthreads, gtid;
  group_coords<CS>(g, gthreads, gtid);
  const uint32_t V = a.V;
  uint4* state = a.ws.state + (size_t)g * V;
  uint32_t* mark = a.ws.mark + (size_t)g * V;
  uint32_t* list0 = a.ws.list0 + (size_t)g * V;
  uint32_t* list1 = a.ws.list1 + (size_t)g * V;
  GroupCtl* ctl = a.ws.ctl + g;
  if (threadIdx.x == 0) { st.n = 0; st.m_tau = INF_BITS; st.lo = INF_BITS; }
  __syncthreads();

  for (;;) {
    if (gtid == 0) ctl->query = atomicAdd(a.next_query, 1u);
    group_sync<CS>();
    const uint32_t q = __ldcg(&ctl->query);
    if (q >= a.n_queries) break;
    const bool single = (a.n_queries == 1);
    uint32_t* chg = a.ws.chg + (size_t)g * V;
    const int sweeps = 0;                            // in-round sweeps are compiled into the whole-grid kernel only
    for (uint32_t v = gtid; v < V; v += gthreads) {
      state[v] = state_inf(); mark[v] = MARK_NONE; chg[v] = 0u;
      if (sweeps) a.ws.ver[v] = 0u;
    }
    group_sync<CS>();

    const uint32_t sf = a.seed_faces[q];
    const uint32_t s0 = a.faces[3 * (size_t)sf], s1 = a.faces[3 * (size_t)sf + 1], s2 = a.faces[3 * (size_t)sf + 2];
    CvpEllProblem prob;
    prob.cor_ptr = a.cor_ptr; prob.cor_idx = a.cor_idx; prob.cor_w = a.cor_w; prob.cost = a.cost; prob.invalid = a.invalid;
    prob.ell_idx = a.ell_idx; prob.ell_w = a.ell_w; prob.ell_geo = a.ell_geo;
    prob.state = state; prob.ext_arr = a.ws.ext + (size_t)g * V; prob.root_arr = a.ws.root + (size_t)g * V; prob.chg = chg;
    prob.pool_w = a.ws.pool + (size_t)g * a.ws.pool_cap; prob.pool = prob.pool_w; prob.pool_cap = a.ws.pool_cap; prob.pool_top = &ctl->pool_top; prob.pool_overflow = &ctl->pool_overflow;
    prob.ver = a.ws.ver; prob.deferred_m = __uint_as_float(INF_BITS); prob.pred = nullptr; prob.dir = nullptr; prob.cut = nullptr; prob.cost_limit = a.cost_limit;
    prob.s0 = s0; prob.s1 = s1; prob.s2 = s2; prob.seed_noexpand = 0; prob.goal_t = ev_normal(__uint_as_float(INF_BITS), 0u);
    prob.prefetch_marks = false;
    float sd[3];
    {
      const uint32_t sv[3] = {s0, s1, s2};
      for (int k = 0; k < 3; ++k) {   // cvp:719-728
        const float dx = a.seed_pos[3 * (size_t)q] - a.pos[3 * (size_t)sv[k]];
        const float dy = a.seed_pos[3 * (size_t)q + 1] - a.pos[3 * (size_t)sv[k] + 1];
        const float dz = a.seed_pos[3 * (size_t)q + 2] - a.pos[3 * (size_t)sv[k] + 2];
        sd[k] = sqrtf(dx * dx + dy * dy + dz * dz);
        const bool noexp = ((double)a.cost[sv[k]] >= a.cost_limit) || (a.invalid && a.invalid[sv[k]]);  // cvp:757,760
        if (noexp) prob.seed_noexpand |= (1u << k);
      }
    }
    const float seed_min = fminf(sd[0], fminf(sd[1], sd[2]));
    const float seed_max = fmaxf(sd[0], fmaxf(sd[1], sd[2]));
    prob.seed_max_d = seed_max;
    uint32_t r0 = 0xffffffffu, r1 = 0xffffffffu, r2 = 0xffffffffu;
    const int has_robot = single && a.robot_face >= 0;
    if (has_robot) {
      r0 = a.faces[3 * (size_t)a.robot_face]; r1 = a.faces[3 * (size_t)a.robot_face + 1]; r2 = a.faces[3 * (size_t)a.robot_face + 2];
    }
    if (gtid == 0) {
      const uint32_t sv[3] = {s0, s1, s2};
      for (int k = 0; k < 3; ++k) {
        state[sv[k]] = make_uint4(__float_as_uint(sd[k]), __float_as_uint(sd[k]), 0u, 0u);
        mark[sv[k]] = MARK_FIXED;
      }
      unsigned int n0 = 0;
      for (int k = 0; k < 3; ++k)
        prob.activate(sv[k], [&](uint32_t x) {
          if (mark[x] == MARK_NONE && prob.eligible(x)) { mark[x] = MARK_CAND; list0[n0++] = x; }
        });
      ctl_reset(ctl, n0, seed_min);
      if (has_robot) {
        int left = 0; const uint32_t rv[3] = {r0, r1, r2};
        for (int k = 0; k < 3; ++k) if (mark[rv[k]] != MARK_FIXED) left++;
        ctl->robot_left = left;
        if (left == 0) {  // robot face == seed face: cutoff armed when the last seed pops (cvp:763-771)
          ctl->goal_ring[0] = __float_as_uint((float)((double)seed_max + a.goal_dist_offset));
          uint32_t sl = sv[0]; float sdl = sd[0];
          for (int k = 1; k < 3; ++k) if (sd[k] > sdl || (sd[k] == sdl && sv[k] > sl)) { sl = sv[k]; sdl = sd[k]; }
          ctl->goal_time[0] = __float_as_uint(sdl); ctl->goal_time[1] = sl; ctl->goal_time[5] = sl;
        }
      }
    }
    group_sync<CS>();
    float delta = a.delta;
    if (has_robot && a.goal_dist_offset < (double)delta) delta = (float)fmax(a.goal_dist_offset, 1e-4);
    run_band_rounds_sub8<CS, false>(prob, ctl, list0, list1, mark, st, delta, gthreads, gtid, has_robot, r0, r1, r2,
                        a.goal_dist_offset, a.cancel_flag, nextafterf(seed_max, __uint_as_float(INF_BITS)), a.max_rounds, sweeps, nullptr, V);
    group_sync<CS>();
    if (a.out_dist) {
      float* od = a.out_dist + (size_t)q * V;
      for (uint32_t v = gtid; v < V; v += gthreads) od[v] = __uint_as_float(state[v].x);
    }
    group_sync<CS>();
  }
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
// The problem object: the workspace group's labels, the goal's seed face sf, the goal cutoff's pop time (not armed: +inf)
// and the outputs (any may be null).
__device__ __forceinline__ void cvp_epilogue_problem(const CvpKernelArgs& a, uint4* state, uint32_t* ext, uint32_t* root, uint32_t* chg,
                                                     uint32_t* pool, GroupCtl* ctl, uint32_t sf, const EvTime& goal_t,
                                                     uint32_t* pred, float* dir, int32_t* cut, CvpProblem& prob) {
  prob.cor_ptr = a.cor_ptr; prob.cor_idx = a.cor_idx; prob.cor_w = a.cor_w; prob.cost = a.cost; prob.invalid = a.invalid;
  prob.state = state; prob.ext_arr = ext; prob.root_arr = root; prob.chg = chg;
  prob.pool_w = pool; prob.pool = pool; prob.pool_cap = a.ws.pool_cap; prob.pool_top = &ctl->pool_top; prob.pool_overflow = &ctl->pool_overflow;
  prob.ver = nullptr; prob.deferred_m = __uint_as_float(INF_BITS); prob.pred = pred; prob.dir = dir; prob.cut = cut; prob.cost_limit = a.cost_limit;
  prob.strict = 0;
  prob.s0 = a.faces[3 * (size_t)sf]; prob.s1 = a.faces[3 * (size_t)sf + 1]; prob.s2 = a.faces[3 * (size_t)sf + 2];
  prob.seed_noexpand = 0;
  prob.goal_t = goal_t;
  const uint32_t sv[3] = {prob.s0, prob.s1, prob.s2};
  for (int k = 0; k < 3; ++k)
    if (((double)a.cost[sv[k]] >= a.cost_limit) || (a.invalid && a.invalid[sv[k]])) prob.seed_noexpand |= (1u << k);
}

// one vertex c of the epilogue (goal: the goal cutoff's potential, +inf when not armed)
__device__ __forceinline__ void cvp_epilogue_vertex(CvpProblem& prob, GroupCtl* ctl, uint32_t sf, float goal, uint32_t c) {
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
  int win = -1; float nd, wu1 = 0, wu2 = 0; EvFull nt;
  if (__float_as_uint(d) != INF_BITS && prob.eligible(c))
    prob.replay(c, __uint_as_float(INF_BITS), goal, 0xfffffff0u /* final labels: nothing is deferred */, nd, nt, win, wu1, wu2);
  prob.write_aux(c, win, wu1, wu2);
}

// k_cvp_batch<CS, true>: the epilogue of goal q over the group's workspace, rows q of out_pred / out_dir / out_cut (each may
// be null).  Out of line: its frame (the replay holds a vertex's faces) does not weigh on the registers of the round loop.
__device__ __noinline__ void batch_fields_epilogue(const CvpKernelArgs& a, const BatchGroup& G, uint32_t q, uint32_t gthreads, uint32_t gtid) {
  const uint32_t V = a.V;
  const size_t row = (size_t)q * V;
  const uint32_t sf = a.seed_faces[q];
  CvpProblem prob;
  cvp_epilogue_problem(a, G.state, G.ext_arr, G.root_arr, G.chg, G.pool, G.ctl, sf, ev_normal(__uint_as_float(INF_BITS), 0u),
                       a.out_pred ? a.out_pred + row : nullptr, a.out_dir ? a.out_dir + row : nullptr, a.out_cut ? a.out_cut + row : nullptr, prob);
  for (uint32_t v = gtid; v < V; v += gthreads) cvp_epilogue_vertex(prob, G.ctl, sf, __uint_as_float(INF_BITS), v);
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
  if (threadIdx.x == 0) { st.n = 0; st.m_tau = INF_BITS; st.lo = INF_BITS; wk.n = 0; wk.ns = 0; }
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
    const uint32_t sf = a.seed_faces[q];
    BatchSeeds sd;
    sd.s0 = a.faces[3 * (size_t)sf]; sd.s1 = a.faces[3 * (size_t)sf + 1]; sd.s2 = a.faces[3 * (size_t)sf + 2]; sd.noexpand = 0;
    float sdist[3];
    {
      const uint32_t sv[3] = {sd.s0, sd.s1, sd.s2};
      for (int k = 0; k < 3; ++k) {   // cvp:719-728
        const float dx = a.seed_pos[3 * (size_t)q] - a.pos[3 * (size_t)sv[k]];
        const float dy = a.seed_pos[3 * (size_t)q + 1] - a.pos[3 * (size_t)sv[k] + 1];
        const float dz = a.seed_pos[3 * (size_t)q + 2] - a.pos[3 * (size_t)sv[k] + 2];
        sdist[k] = sqrtf(dx * dx + dy * dy + dz * dz);
        if (((double)a.cost[sv[k]] >= a.cost_limit) || (a.invalid && a.invalid[sv[k]])) sd.noexpand |= (1u << k);  // cvp:757,760
      }
    }
    const float seed_min = fminf(sdist[0], fminf(sdist[1], sdist[2]));
    sd.seed_max = fmaxf(sdist[0], fmaxf(sdist[1], sdist[2]));
    if (gtid == 0) {
      const uint32_t sv[3] = {sd.s0, sd.s1, sd.s2};
      for (int k = 0; k < 3; ++k) {
        G.state[sv[k]] = make_uint4(__float_as_uint(sdist[k]), __float_as_uint(sdist[k]), 0u, 0u);
        G.mark[sv[k]] = MARK_FIXED;
      }
      unsigned int n0 = 0;
      for (int k = 0; k < 3; ++k) {
        const uint32_t kb = a.cor_ptr[sv[k]], ke = a.cor_ptr[sv[k] + 1];
        for (uint32_t kk = kb; kk < ke; ++kk) {
          const int4 ix = a.cor_idx[kk];
          const uint32_t xs[2] = {(uint32_t)ix.x, (uint32_t)ix.y};
          for (int t = 0; t < 2; ++t) {
            const uint32_t x = xs[t];
            if (G.mark[x] == MARK_NONE && !(a.invalid && a.invalid[x]) && !((double)a.cost[x] >= a.cost_limit)) { G.mark[x] = MARK_CAND; list0[n0++] = x; }
          }
        }
      }
      ctl_reset(ctl, n0, seed_min);
      if constexpr (MATRIX) ctl->targets_left = (int)a.tg.distinct;
    }
    group_sync<CS>();
    if constexpr (MATRIX) {
      count_targets_done_at_init(a.tg, ctl, G.mark, V, gthreads, gtid, [&](uint32_t v) {   // candidates: k_cvp_batch's activation test
        return !(a.invalid && a.invalid[v]) && !((double)a.cost[v] >= a.cost_limit);
      });
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
__global__ void __launch_bounds__(512, MNB_GRID_MINBLOCKS) k_cvp_grid(const CvpKernelArgs a) {
  __shared__ Stage st;
  __shared__ SweepStage sws;
  uint32_t g, gthreads, gtid;
  group_coords<0>(g, gthreads, gtid);
  const uint32_t V = a.V;
  uint4* state = a.ws.state; uint32_t* mark = a.ws.mark; uint32_t* list0 = a.ws.list0; uint32_t* list1 = a.ws.list1;
  GroupCtl* ctl = a.ws.ctl;
  if (threadIdx.x == 0) { st.n = 0; st.m_tau = INF_BITS; st.lo = INF_BITS; sws.dn[0] = 0; sws.dn[1] = 0; }
  __syncthreads();
  for (uint32_t v = gtid; v < V; v += gthreads) { state[v] = state_inf(); mark[v] = MARK_NONE; a.ws.chg[v] = 0u; a.ws.ver[v] = 0u; }
  group_sync<0>(ctl->barrier);
  const uint32_t sf = a.seed_faces[0];
  const uint32_t s0 = a.faces[3 * (size_t)sf], s1 = a.faces[3 * (size_t)sf + 1], s2 = a.faces[3 * (size_t)sf + 2];
  CvpEllProblem prob;
  prob.cor_ptr = a.cor_ptr; prob.cor_idx = a.cor_idx; prob.cor_w = a.cor_w; prob.cost = a.cost; prob.invalid = a.invalid;
  prob.ell_idx = a.ell_idx; prob.ell_w = a.ell_w; prob.ell_geo = a.ell_geo;
  prob.state = state; prob.ext_arr = a.ws.ext; prob.root_arr = a.ws.root; prob.chg = a.ws.chg;
  prob.pool_w = a.ws.pool; prob.pool = prob.pool_w; prob.pool_cap = a.ws.pool_cap; prob.pool_top = &ctl->pool_top; prob.pool_overflow = &ctl->pool_overflow;
  prob.ver = a.ws.ver; prob.deferred_m = __uint_as_float(INF_BITS); prob.pred = nullptr; prob.dir = nullptr; prob.cut = nullptr; prob.cost_limit = a.cost_limit;
  prob.s0 = s0; prob.s1 = s1; prob.s2 = s2; prob.seed_noexpand = 0; prob.goal_t = ev_normal(__uint_as_float(INF_BITS), 0u);
  prob.prefetch_marks = true;
  float sd[3];
  {
    const uint32_t sv[3] = {s0, s1, s2};
    for (int k = 0; k < 3; ++k) {   // cvp:719-728
      const float dx = a.seed_pos[0] - a.pos[3 * (size_t)sv[k]];
      const float dy = a.seed_pos[1] - a.pos[3 * (size_t)sv[k] + 1];
      const float dz = a.seed_pos[2] - a.pos[3 * (size_t)sv[k] + 2];
      sd[k] = sqrtf(dx * dx + dy * dy + dz * dz);
      const bool noexp = ((double)a.cost[sv[k]] >= a.cost_limit) || (a.invalid && a.invalid[sv[k]]);
      if (noexp) prob.seed_noexpand |= (1u << k);
    }
  }
  const float seed_min = fminf(sd[0], fminf(sd[1], sd[2]));
  const float seed_max = fmaxf(sd[0], fmaxf(sd[1], sd[2]));
  prob.seed_max_d = seed_max;
  uint32_t r0 = 0xffffffffu, r1 = 0xffffffffu, r2 = 0xffffffffu;
  const int has_robot = a.robot_face >= 0;
  if (has_robot) {
    r0 = a.faces[3 * (size_t)a.robot_face]; r1 = a.faces[3 * (size_t)a.robot_face + 1]; r2 = a.faces[3 * (size_t)a.robot_face + 2];
  }
  if (gtid == 0) {
    const uint32_t sv[3] = {s0, s1, s2};
    for (int k = 0; k < 3; ++k) { state[sv[k]] = make_uint4(__float_as_uint(sd[k]), __float_as_uint(sd[k]), 0u, 0u); mark[sv[k]] = MARK_FIXED; }
    unsigned int n0 = 0;
    for (int k = 0; k < 3; ++k)
      prob.activate(sv[k], [&](uint32_t x) {
        if (mark[x] == MARK_NONE && prob.eligible(x)) { mark[x] = MARK_CAND; list0[n0++] = x; }
      });
    ctl_reset(ctl, n0, seed_min);
    if (has_robot) {
      int left = 0; const uint32_t rv[3] = {r0, r1, r2};
      for (int k = 0; k < 3; ++k) if (mark[rv[k]] != MARK_FIXED) left++;
      ctl->robot_left = left;
      if (left == 0) {
        ctl->goal_ring[0] = __float_as_uint((float)((double)seed_max + a.goal_dist_offset));
        uint32_t sl = sv[0]; float sdl = sd[0];
        for (int k = 1; k < 3; ++k) if (sd[k] > sdl || (sd[k] == sdl && sv[k] > sl)) { sl = sv[k]; sdl = sd[k]; }
        ctl->goal_time[0] = __float_as_uint(sdl); ctl->goal_time[1] = sl; ctl->goal_time[5] = sl;
      }
    }
  }
  group_sync<0>(ctl->barrier);
  const float delta = a.delta;      // not clamped to goal_dist_offset: the engine caps settling instead (settle_cap)
  // in-round sweeps pay off once the band is several dependency hops deep; 12 were measured best on the 5M terrain
  int sweeps = a.sweeps;
  if (sweeps < 0) sweeps = delta < 2.8f * a.hop ? 0 : min(12, (int)(delta / a.hop));
  run_band_rounds_sub8<0, true>(prob, ctl, list0, list1, mark, st, delta, gthreads, gtid, has_robot, r0, r1, r2,
                          a.goal_dist_offset, a.cancel_flag, nextafterf(seed_max, __uint_as_float(INF_BITS)), a.max_rounds, sweeps, &sws, V);
  group_sync<0>(ctl->barrier);
  if (a.out_dist)
    for (uint32_t v = gtid; v < V; v += gthreads) a.out_dist[v] = __uint_as_float(state[v].x);
}

// the epilogue of a single plan (cvp_epilogue_problem above), one thread per vertex; the goal cutoff is the plan's
__global__ void __launch_bounds__(256) k_cvp_epilogue(const CvpKernelArgs a, GroupCtl* ctl) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.V) return;
  const uint32_t sf = a.seed_faces[0];
  EvTime goal_t;
  goal_t.a1 = __uint_as_float(ctl->goal_time[0]); goal_t.root = ctl->goal_time[1]; goal_t.a2 = __uint_as_float(ctl->goal_time[2]);
  goal_t.a3 = __uint_as_float(ctl->goal_time[3]); goal_t.ext = ctl->goal_time[4]; goal_t.self = ctl->goal_time[5];
  CvpProblem prob;
  cvp_epilogue_problem(a, a.ws.state, a.ws.ext, a.ws.root, a.ws.chg, a.ws.pool, ctl, sf, goal_t, a.out_pred, a.out_dir, a.out_cut, prob);
  cvp_epilogue_vertex(prob, ctl, sf, __uint_as_float(ctl->goal_bits), c);
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
  const uint4* ell_adj; int sweeps; float hop;   // whole-grid kernel only
};

template <int CS>
__global__ void __launch_bounds__(512, 1) k_dijkstra(const DijkstraKernelArgs a) {
  __shared__ Stage st;
  uint32_t g, gthreads, gtid;
  group_coords<CS>(g, gthreads, gtid);
  const uint32_t V = a.V;
  uint4* state = a.ws.state;
  uint32_t* mark = a.ws.mark; uint32_t* list0 = a.ws.list0; uint32_t* list1 = a.ws.list1;
  GroupCtl* ctl = a.ws.ctl;
  if (threadIdx.x == 0) { st.n = 0; st.m_tau = INF_BITS; st.lo = INF_BITS; }
  __syncthreads();
  for (uint32_t v = gtid; v < V; v += gthreads) { state[v] = state_inf(); mark[v] = MARK_NONE; a.out_pred[v] = v; }
  group_sync<CS>(ctl->barrier);
  DijkstraProblem prob;
  prob.adj_ptr = a.adj_ptr; prob.adj_nw = a.adj_nw; prob.cost = a.cost; prob.invalid = a.invalid;
  prob.state = state; prob.pred = a.out_pred; prob.cost_limit = a.cost_limit; prob.deferred_m = __uint_as_float(INF_BITS);
  const int has_robot = a.robot_vertex >= 0;
  const uint32_t rv = has_robot ? (uint32_t)a.robot_vertex : 0xffffffffu;
  if (gtid == 0) {
    state[a.seed_vertex] = make_uint4(0u, 0u, 0u, 0u);     // dijkstra:276 (d = 0, tau = 0)
    mark[a.seed_vertex] = MARK_FIXED;
    unsigned int n0 = 0;
    prob.activate(a.seed_vertex, [&](uint32_t x) {
      if (mark[x] == MARK_NONE && prob.eligible(x)) { mark[x] = MARK_CAND; list0[n0++] = x; }
    });
    ctl_reset(ctl, n0, 0.0f);
    if (has_robot) ctl->robot_left = 1;
  }
  group_sync<CS>();
  float delta = a.delta;
  if (has_robot && a.goal_dist_offset < (double)delta) delta = (float)fmax(a.goal_dist_offset, 1e-4);
  run_band_rounds<CS>(prob, ctl, list0, list1, mark, st, delta, gthreads, gtid, has_robot, rv, rv, rv,
                      a.goal_dist_offset, a.cancel_flag, 1e-30f, a.max_rounds);
  group_sync<CS>();
  for (uint32_t v = gtid; v < V; v += gthreads) a.out_dist[v] = __uint_as_float(state[v].x);
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
  if (threadIdx.x == 0) { st.n = 0; st.m_tau = INF_BITS; st.lo = INF_BITS; }
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
    const uint32_t s = a.seeds[q];
    if (gtid == 0) {
      label[s] = 0.0f;                                         // dijkstra:276
      mark[s] = MARK_FIXED;
      unsigned int n0 = 0;
      prob.activate(s, [&](uint32_t x) {
        if (mark[x] == MARK_NONE && prob.eligible(x)) { mark[x] = MARK_CAND; list0[n0++] = x; }
      });
      ctl_reset(ctl, n0, 0.0f);
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

// Single Dijkstra plan on the whole GPU: 8 lanes per candidate (one edge each), wide band + in-round sweeps,
// same engine instance as k_cvp_grid.
__global__ void __launch_bounds__(512, 1) k_dijkstra_grid(const DijkstraKernelArgs a) {
  __shared__ Stage st;
  __shared__ SweepStage sws;
  uint32_t g, gthreads, gtid;
  group_coords<0>(g, gthreads, gtid);
  const uint32_t V = a.V;
  uint4* state = a.ws.state;
  uint32_t* mark = a.ws.mark; uint32_t* list0 = a.ws.list0; uint32_t* list1 = a.ws.list1;
  GroupCtl* ctl = a.ws.ctl;
  if (threadIdx.x == 0) { st.n = 0; st.m_tau = INF_BITS; st.lo = INF_BITS; sws.dn[0] = 0; sws.dn[1] = 0; }
  __syncthreads();
  for (uint32_t v = gtid; v < V; v += gthreads) { state[v] = state_inf(); mark[v] = MARK_NONE; a.out_pred[v] = v; a.ws.ver[v] = 0u; }
  group_sync<0>(ctl->barrier);
  DijkstraEllProblem prob;
  prob.adj_ptr = a.adj_ptr; prob.adj_nw = a.adj_nw; prob.cost = a.cost; prob.invalid = a.invalid;
  prob.state = state; prob.pred = a.out_pred; prob.cost_limit = a.cost_limit; prob.deferred_m = __uint_as_float(INF_BITS);
  prob.strict = 0; prob.ell_adj = a.ell_adj; prob.ver = a.ws.ver;
  const int has_robot = a.robot_vertex >= 0;
  const uint32_t rv = has_robot ? (uint32_t)a.robot_vertex : 0xffffffffu;
  if (gtid == 0) {
    state[a.seed_vertex] = make_uint4(0u, 0u, 0u, 0u);     // dijkstra:276 (d = 0, tau = 0)
    mark[a.seed_vertex] = MARK_FIXED;
    unsigned int n0 = 0;
    prob.activate(a.seed_vertex, [&](uint32_t x) {
      if (mark[x] == MARK_NONE && prob.eligible(x)) { mark[x] = MARK_CAND; list0[n0++] = x; }
    });
    ctl_reset(ctl, n0, 0.0f);
    if (has_robot) ctl->robot_left = 1;
  }
  group_sync<0>(ctl->barrier);
  const float delta = a.delta;      // not clamped to goal_dist_offset: the engine caps settling instead (settle_cap)
  int sweeps = a.sweeps;
  if (sweeps < 0) sweeps = delta < 2.8f * a.hop ? 0 : min(15, (int)(delta / a.hop));
  run_band_rounds_sub8<0, true>(prob, ctl, list0, list1, mark, st, delta, gthreads, gtid, has_robot, rv, rv, rv,
                                a.goal_dist_offset, a.cancel_flag, 1e-30f, a.max_rounds, sweeps, &sws, V);
  group_sync<0>(ctl->barrier);
  for (uint32_t v = gtid; v < V; v += gthreads) a.out_dist[v] = __uint_as_float(state[v].x);
}
