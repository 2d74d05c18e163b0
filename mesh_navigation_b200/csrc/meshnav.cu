// libmeshnav_b200.so -- C ABI (include/meshnav_b200.h) over the sm_90a kernels.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -fmad=false -std=c++17
//             -Xcompiler -fPIC -shared -o libmeshnav_b200.so meshnav.cu
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <functional>
#include <map>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/meshnav_b200.h"
#include "band_engine.cuh"
#include "problems.cuh"
#include "topology.hpp"

using namespace mnb;

#include "launch.cuh"
#include "kernels_maps.cuh"
#include "kernels_wavefront.cuh"
#include "kernels_layers.cuh"
#include "kernels_field.cuh"
#include "kernels_updates.cuh"
#include "kernels_raycast.cuh"
#include "kernels_infl_repair.cuh"

// mnb_inflation_repair runs the whole-map wave when more than this share of the old footprint lies in affected clusters:
// the local path pays its O(V) passes on top of the wave and, when a new footprint reaches an unaffected cluster, a second
// pass over everything affected.  On the 5 M bench map (DESIGN §5, H100 at 700 W) the local path took 1.1 ms against
// 6.6 ms for the full call at a share of 0.0002, 5.4 against 6.7 ms at 0.28 and 10.3 against 6.6 ms at 0.70.
constexpr double INFL_REPAIR_MAX_SHARE = 0.5;

// default band width of the batched Dijkstra planner in mean edge weights: on the 1 M terrain with 1024 goals 1.5 w was
// fastest of 1 - 10 w (DESIGN §5)
constexpr float DIJKSTRA_BATCH_DELTA_W = 1.5f;
// GridStage slots per CTA of the whole-grid single-plan kernels (k_cvp_grid, k_dijkstra_grid), fewer if the device's
// opt-in shared memory per block holds fewer.  Measured on the 5 M bench plan (tools/gpu_sweep_slots.py; H100 80GB HBM3,
// 700 W, 1980 MHz; median of 5 plans, L2 flushed): at the best band and sweep count of each, k_cvp_grid + epilogue took
// 37.1 ms with 1024 slots (20 w, 12 sweeps), 34.6 ms with 2048 (40 w, 24), 35.1 ms with 3072 (60 w, 48), 35.9 ms with 4096
// (40 w, 24) and 39.1 ms with 6144 (60 w, 48).  More slots take fewer rounds (117 at 2048, 75 at 3072), but the shared
// memory they take (30 B per slot) comes out of the L1 that caches the ELL rows the sweeps read: at 20 w the same plan
// costs 37.1 / 37.2 / 37.9 / 38.8 / 42.2 ms from 1024 to 6144 slots.  2048 slots (60 KB) is the trade-off.
constexpr uint32_t GRID_SLOTS_DEFAULT = 2048;
// single-plan band widths in mean edge weights w (install_weights): 40 w measured best for both kernels at 2048 slots
// (CVP: 37.2 / 35.3 / 34.6 / 38.2 ms at 20 / 30 / 40 / 60 w with their best sweep counts; Dijkstra: 12.0 / 11.1 / 11.0 ms at
// 25 / 40 / 60 w, where 60 w needs 24 sweeps and 40 w keeps the 15 of the sweep rule)
constexpr float GRID_BAND_W = 40.0f;
// static shared memory of the whole-grid kernels (GridStage's counters and the main pass's queue length) is far below this
constexpr size_t GRID_STATIC_SMEM_ROOM = 1024;

// ============================================================================
// host side
// ============================================================================
// One device array and its owner: a capacity in elements that only grows (reserve) and a release in the destructor.  It
// converts to T*, so launches and copies read as with a raw pointer.  A failed reserve leaves the buffer empty (null,
// capacity 0), never a null pointer under the capacity of the array it replaced.
template <class T>
struct DeviceBuffer {
  T* p = nullptr;
  size_t cap = 0;
  DeviceBuffer() = default;
  DeviceBuffer(DeviceBuffer&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DeviceBuffer& operator=(DeviceBuffer&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
  ~DeviceBuffer() { if (p) cudaFree(p); }
  operator T*() const { return p; }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    const cudaError_t e = cudaMalloc((void**)&p, n * sizeof(T));
    if (e == cudaSuccess) cap = n; else p = nullptr;
    return e;
  }
};

// Ray caster over the faces (kernels_raycast.cuh; built on first use) + state of the obstacle layer.  A default-constructed
// value is "not built": free_raycaster assigns one.
struct RayCasterState {
  bool bvh_valid = false; float bvh_eps = 0.0f;
  DeviceBuffer<float4> bvh_lo, bvh_hi; DeviceBuffer<uint32_t> bvh_parent, bvh_order; DeviceBuffer<unsigned int> bvh_visits, bvh_scene;   // the arrays of RayBvh (ray_bvh)
  DeviceBuffer<unsigned int> d_ray_overflow;
  DeviceBuffer<float> d_ray_in, d_ray_out;      // staging of host-pointer inputs / outputs of the ray calls
  DeviceBuffer<uint8_t> d_obst_now, d_obst_mask; DeviceBuffer<float> d_obst_member, d_obst_member_chg;
  DeviceBuffer<uint32_t> d_obst_list;
};

// the arrays of WaveWorkspace / DijkstraBatchWorkspace (wave_workspace, dijkstra_workspace fill the kernels' views)
struct WaveBuffers {
  DeviceBuffer<uint4> state, skipw;
  DeviceBuffer<uint32_t> ext, root, pool, last_eval, dirty, chg, ver, mark, list0, list1;
  DeviceBuffer<GroupCtl> ctl;
};
struct DijkstraBatchBuffers { DeviceBuffer<float> label; DeviceBuffer<uint32_t> mark, list0, list1; DeviceBuffer<GroupCtl> ctl; };
// one resident wave of mnb_cvp_batch_replan: its goal (seed face, seed position bits), whether it holds that goal's wave of
// the store's costs and cost limit, and its own allocation (ReplanSlot, kernels_wavefront.cuh) -- growing the store moves
// no slot
struct BatchReplanSlot {
  uint32_t face = 0, pos[3] = {0, 0, 0};
  bool valid = false;
  DeviceBuffer<uint8_t> mem;
};

// Everything that is sized by the mesh or computed from it, with the flags and counters that describe it.  A
// default-constructed value is "no mesh": free_mesh assigns one, so a buffer declared here needs no other bookkeeping.
struct MeshState : RayCasterState {
  uint32_t V = 0, F = 0, E = 0;
  size_t NC = 0, NA = 0;
  DeviceBuffer<float> d_pos; DeviceBuffer<uint32_t> d_faces, d_edges;
  DeviceBuffer<uint32_t> d_cor_ptr; DeviceBuffer<int4> d_cor_idx; DeviceBuffer<uint4> d_cor_eid; DeviceBuffer<uint32_t> d_face_cor;
  DeviceBuffer<float4> d_cor_w, d_cor_wd;
  DeviceBuffer<int4> d_ell_idx; DeviceBuffer<uint4> d_ell_eid; DeviceBuffer<float4> d_ell_w, d_ell_wd; DeviceBuffer<double4> d_ell_geo;
  DeviceBuffer<uint32_t> d_adj_ptr, d_adj_nbr, d_adj_eid; DeviceBuffer<uint2> d_adj_nw; DeviceBuffer<uint4> d_ell_adj;
  DeviceBuffer<float> d_edge_dist, d_edge_w, d_cost; DeviceBuffer<uint8_t> d_invalid;
  DeviceBuffer<double> d_wsum;       // sums of install_weights (mnb_ctx::w_mean)
  bool costs_set = false;
  // workspace
  uint32_t ws_groups = 0;
  WaveBuffers ws;
  uint32_t dws_groups = 0;       // the batched Dijkstra planner's own workspace (k_dijkstra_batch)
  DijkstraBatchBuffers dws;
  bool dws_marks_clean = false;  // every mark of dws is MARK_NONE: the repair kernel leaves them so, the batch kernel does not
  DeviceBuffer<uint32_t> d_batch_pred;    // its predecessor rows in host-pointer mode (and mnb_cvp_batch_fields')
  DeviceBuffer<float> d_batch_dir;        // mnb_cvp_batch_fields' direction and cutting-face rows in host-pointer mode
  DeviceBuffer<int32_t> d_batch_cut;
  // scratch outputs for host-pointer mode
  DeviceBuffer<float> d_out_dist, d_out_dir, d_out_cost; DeviceBuffer<uint32_t> d_out_pred; DeviceBuffer<int32_t> d_out_cut;
  // target vertices of the cost-matrix calls: the caller's list and the bitmap of the distinct ones (V/32 + 1 words)
  DeviceBuffer<uint32_t> d_targets, d_target_bits;
  // changed vertices of a field repair: the distinct ones, their bitmap (V/32 + 1 words), the per-group log lengths
  DeviceBuffer<uint32_t> d_repair_chg, d_repair_bits; DeviceBuffer<unsigned int> d_repair_log_n;
  DeviceBuffer<float> d_face_normals, d_vertex_normals; DeviceBuffer<uint8_t> d_border;
  DeviceBuffer<float> d_layer_costs, d_layer_combined, d_clearance; DeviceBuffer<uint8_t> d_layer_mask;
  DeviceBuffer<float4> d_pos4, d_vn4; DeviceBuffer<uint32_t> d_nbr8;     // packed copies for the prefetching layer walk
  DeviceBuffer<unsigned int> d_overflow;
  // device-resident result of the last single CVP plan (for mnb_cvp_backtrack)
  const uint32_t* last_pred = nullptr; const float* last_dir = nullptr; const int32_t* last_cut = nullptr;
  uint32_t last_seed_face = 0; float last_seed_pos[3] = {0, 0, 0}; bool last_valid = false;
  // generation of the installed costs: mnb_set_costs and mnb_compute_edge_weights start a new one (mnb_set_mesh a new
  // MeshState), mnb_update_vertex_costs does not -- a replan may resume across it
  uint64_t cost_gen = 0;
  // mnb_cvp_replan: the resident wave of the last successful replan in its own workspace (labels, side arrays, level pool,
  // marks, lists, sweep versions, control block; allocated by the first replan) and what it was computed for
  WaveBuffers rw;
  bool epi_in_rw = false;        // the last single plan's epilogue ran on rw (mnb_debug_get_epilogue_csr), not on ws
  bool rw_valid = false; uint32_t rw_seed_face = 0, rw_seed_pos[3] = {0, 0, 0}; uint64_t rw_cost_limit = 0, rw_cost_gen = 0;
  uint32_t rw_pool_top = 0;
  DeviceBuffer<uint32_t> d_replan_chg, d_replan_t0;      // the changed list of a replan, T0 and the block minima of its reduction
  // mnb_cvp_batch_replan: the resident slots (at most one per goal), the cost limit and cost generation their waves were
  // computed for, the goal table and the T0 minima of a call
  std::vector<BatchReplanSlot> brs;
  uint64_t brs_cost_limit = 0, brs_cost_gen = 0;
  DeviceBuffer<BatchReplanGoal> d_brs_goals; DeviceBuffer<uint32_t> d_brs_minima;
  DeviceBuffer<float> d_path_pos; DeviceBuffer<uint32_t> d_path_face; DeviceBuffer<int32_t> d_bt_result;
  DeviceBuffer<uint32_t> d_bt_spill_list, d_bt_spill_key;   // F each: k_backtrack's unbounded face search (first walk that needs it)
  DeviceBuffer<uint8_t> d_infl_invalid;
  // repulsive vector field of the last inflation (InflationLayer::vector_map_ / distances_)
  bool infl_labels_valid = false, infl_had_invalid = false, infl_field_valid = false, repulsive_on = false;
  mnb_inflation_params infl_params{}; uint64_t infl_rounds = 0;
  DeviceBuffer<float> d_infl_vec, d_infl_dist; DeviceBuffer<int4> d_infl_src; DeviceBuffer<unsigned int> d_infl_flag;
  bool infl_field_resident = false;  // the field is the answer of mnb_inflation_vector_map as it stands (a repair kept it)
  // inflation repair: infl_resident = distances_, riskiness, the lethal set (mnb_ctx::d_lethals, infl_n_lethals) and the
  // invalid mask of the last inflation are on the device.  The staging of the next set and mask, the cluster ids of the
  // footprint (built by the first repair after a whole-map wave), four bitmaps of V/32 + 1 words (old lethals, new
  // lethals, affected clusters, changed riskiness), the seed and region lists and the counters of k_infl_*
  bool infl_resident = false, infl_cid_valid = false; uint32_t infl_n_lethals = 0;
  DeviceBuffer<uint32_t> d_infl_lethals_next; DeviceBuffer<uint8_t> d_infl_invalid_next;
  DeviceBuffer<uint32_t> d_infl_cid, d_infl_bits, d_infl_seeds, d_infl_region; DeviceBuffer<unsigned int> d_infl_cnt;
  // incremental updates
  DeviceBuffer<float> d_prev_risk; bool prev_risk_valid = false;     // riskiness map of the previous inflation (NaN = no entry)
  DeviceBuffer<uint32_t> d_upd_ids; DeviceBuffer<float> d_upd_costs;
  DeviceBuffer<uint32_t> d_upd_stamp; uint32_t upd_call = 0;      // change-set membership stamps of mnb_update_vertex_costs
  DeviceBuffer<uint32_t> d_changed; DeviceBuffer<unsigned int> d_tile_count, d_total;
};

// The mesh state (replaced as a whole by mnb_set_mesh) and what lives as long as the context: stream, events, the staging
// that is sized by a call and not by the mesh, the tuning.  Arrays one call needs and the next does not are locals of it.
struct mnb_ctx : MeshState {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  int ptr_mode = MNB_PTR_HOST;
  int sm_count = 0;
  HostTopology topo;
  bool has_invalid = false;
  bool adj_dirty = true;       // the Dijkstra planner's weight tables (adj_nw, ell_adj) are rebuilt on its first call after new weights
  DeviceBuffer<unsigned int> d_next_query;
  int* h_cancel = nullptr; int* d_cancel = nullptr;
  DeviceBuffer<uint32_t> d_seed_faces, d_lethals; DeviceBuffer<float> d_seed_pos;
  // tuning
  float delta = 0.3f; int cluster = -1 /* -1: whole-grid cooperative kernel for single plans */; int batch_cluster = 0 /* 0: chosen per call from the goal count */; int threads = 512;
  int grid_blocks_per_sm = 0;
  uint32_t grid_slots = 0;     // GridStage slots per CTA of the whole-grid kernels (mnb_debug_set_sweep_slots); set by mnb_create
  uint32_t grid_slots_max = 0; // as many as the device's opt-in shared memory per block holds (at most GRID_SLOTS_MAX)
  size_t grid_smem_set[3] = {0, 0, 0};   // dynamic shared memory the three whole-grid kernels were last checked and set up for
  int infl_skip_clean = 1;     // clean-candidate skip of the inflation wave (mnb_debug_set_infl_skip(ctx, 0) turns it off)
  int layers_walk = LAYERS_WALK_PF16;   // neighbourhood walk of k_layers: LAYERS_WALK_LOCAL (thread-local seen-set),
                                        // LAYERS_WALK_PF32 / LAYERS_WALK_PF16 (prefetching walk, 32-bit / compact seen-set).
                                        // Chosen per mesh by mnb_set_mesh unless fixed by mnb_debug_set_layers_smem.
  bool layers_explicit = false;
  uint32_t replan_pool_room = 0;   // level-pool words a resumed replan wave may add (mnb_debug_set_replan_pool_room; 0 = the pool's)
  uint32_t brs_max_slots = 0xffffffffu;   // cap on the resident slots of mnb_cvp_batch_replan (mnb_debug_set_batch_replan_slots)
  int sweeps = -1;             // in-round sweeps of the whole-grid single plans (mnb_debug_set_sweeps); -1 = derived from the band width
  int cvp_epilogue = 0;        // single-plan epilogue (mnb_debug_set_cvp_epilogue): 0 row replay where it applies, 1 CSR replay for all
  float grid_delta = 1.8f;     // band width of the whole-grid single-plan kernel (wide band + in-round sweeps)
  float dijkstra_grid_delta = 3.0f;
  float dijkstra_batch_delta = 0.18f;
  // The band widths above are potentials, i.e. multiples of the edge weights: unless the caller fixed them (mnb_set_tuning
  // with band_delta > 0) they follow the mean finite edge weight w of the installed weights -- 2.5 w for batches, 20 w for a
  // single CVP or Dijkstra plan (GRID_BAND_W), less on maps above ~9 M vertices, DIJKSTRA_BATCH_DELTA_W w for
  // Dijkstra batches (install_weights); one dependency hop is
  // ~1.35 w (the in-round sweeps are counted in hops).  On the 0.1 m bench meshes (w = 0.118) that is 0.3 / 2.4 / 3.0 m, the values
  // the kernels were tuned with.
  bool delta_explicit = false; float w_mean = 0.0f;
  mnb_stats stats{};
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

#define CK(call)                                                                   \
  do {                                                                             \
    cudaError_t e_ = (call);                                                       \
    if (e_ != cudaSuccess) {                                                       \
      ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);               \
      return MNB_E_CUDA;                                                           \
    }                                                                              \
  } while (0)

// The caller's arrays of one call in the pointer mode (mnb_set_pointer_mode).  In device-pointer mode the kernels get the
// caller's arrays.  In host-pointer mode they get device staging: in() copies an input there when it is declared, out()
// queues the copy of an output back, and copy_back() issues the copies queued so far after the launch, in the order the
// outputs were declared, on ctx->stream.  A DeviceBuffer staging is reserved only when it is used; a raw one is the
// caller's to reserve.  NULL arrays stay NULL, except that needed() falls back to the staging in both modes for an
// output the call reads itself.  The first error stops all further work; status() reports it.
class CallerArrays {
 public:
  explicit CallerArrays(mnb_ctx* ctx) : stream_(ctx->stream), dev_(ctx->ptr_mode == MNB_PTR_DEVICE) {}
  bool device() const { return dev_; }
  cudaError_t status() const { return err_; }

  template <class T> const T* in(const T* caller, T* staging, size_t n) {
    if (!caller || dev_) return caller;
    return ok() && run(cudaMemcpyAsync(staging, caller, sizeof(T) * n, cudaMemcpyHostToDevice, stream_)) ? staging : nullptr;
  }
  template <class T> const T* in(const T* caller, DeviceBuffer<T>& staging, size_t n) {
    if (!caller || dev_) return caller;
    return ok() && run(staging.reserve(n)) ? in(caller, staging.p, n) : nullptr;
  }
  // an output of n elements; with `late` it has n * *late elements, read when copy_back() runs (a list whose length
  // the call reads back)
  template <class T> T* out(T* caller, T* staging, size_t n, const uint32_t* late = nullptr) {
    if (!caller || dev_) return caller;
    if (!ok()) return nullptr;
    queued_.push_back(Copy{caller, staging, sizeof(T), n, late});
    return staging;
  }
  template <class T> T* out(T* caller, DeviceBuffer<T>& staging, size_t n) {
    if (!caller || dev_) return caller;
    return ok() && run(staging.reserve(n)) ? out(caller, staging.p, n) : nullptr;
  }
  template <class T> T* needed(T* caller, T* staging, size_t n, const uint32_t* late = nullptr) {
    return caller ? out(caller, staging, n, late) : staging;
  }
  template <class T> T* inout(T* caller, DeviceBuffer<T>& staging, size_t n) {
    return in((const T*)caller, staging, n) ? out(caller, staging.p, n) : nullptr;
  }
  cudaError_t copy_back() {
    for (const Copy& c : queued_) {
      const size_t n = c.late ? (size_t)*c.late * c.n : c.n;
      if (n && !run(cudaMemcpyAsync(c.dst, c.src, c.elem * n, cudaMemcpyDeviceToHost, stream_))) break;
    }
    queued_.clear();
    return err_;
  }
  // copies between the caller's arrays and context arrays in either mode
  template <class T> cudaError_t copy_in(T* dst, const T* caller, size_t n) {
    return cudaMemcpyAsync(dst, caller, sizeof(T) * n, dev_ ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, stream_);
  }
  template <class T> cudaError_t copy_out(T* caller, const T* src, size_t n) {
    return cudaMemcpyAsync(caller, src, sizeof(T) * n, dev_ ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, stream_);
  }

 private:
  struct Copy { void* dst; const void* src; size_t elem, n; const uint32_t* late; };
  bool ok() const { return err_ == cudaSuccess; }
  bool run(cudaError_t e) { err_ = e; return ok(); }
  cudaStream_t stream_;
  bool dev_;
  cudaError_t err_ = cudaSuccess;
  std::vector<Copy> queued_;
};

static void free_raycaster(mnb_ctx* c) { static_cast<RayCasterState&>(*c) = RayCasterState{}; }
static void free_mesh(mnb_ctx* c) { static_cast<MeshState&>(*c) = MeshState{}; }

// stats of a call that is not a wavefront (finish_stats): the time between ev0 and ev1, once the stream has synchronised
static void simple_stats(mnb_ctx* ctx, uint64_t launches, uint64_t settled) {
  float ms = 0; cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
  ctx->stats = mnb_stats{}; ctx->stats.kernel_ms = ms; ctx->stats.kernel_launches = launches; ctx->stats.settled = settled;
}

// level pool (band_engine.cuh): pop times with more than 3 cascade levels keep their tails here; 2 words per vertex
// hold the deepest flooded pockets randomised testing has produced with room to spare; exhaustion is reported
static uint32_t ws_pool_cap(uint32_t V) { return (uint32_t)std::min<size_t>(std::max<size_t>(65536, 2 * (size_t)V), 0x7fffffffu); }
// device bytes of one group of the wavefront workspace (ensure_workspace): two 16-byte and six 4-byte words per vertex,
// the level pool and the GroupCtl -- 64 bytes per vertex on large maps
static size_t ws_bytes_per_group(uint32_t V) {
  return (size_t)V * (2 * sizeof(uint4) + 6 * sizeof(uint32_t)) + (size_t)ws_pool_cap(V) * sizeof(uint32_t) + sizeof(GroupCtl);
}

static int32_t ensure_workspace(mnb_ctx* ctx, uint32_t groups) {
  if (groups <= ctx->ws_groups) return MNB_OK;
  WaveBuffers& w = ctx->ws;
  w = WaveBuffers{};         // the smaller workspace goes first: batch_shape has counted its bytes as available
  ctx->ws_groups = 0;
  const size_t n = (size_t)groups * ctx->V, V = ctx->V;
  CK(w.state.reserve(n)); CK(w.ext.reserve(n)); CK(w.skipw.reserve(n)); CK(w.root.reserve(n)); CK(w.last_eval.reserve(V)); CK(w.dirty.reserve(V)); CK(w.chg.reserve(n)); CK(w.ver.reserve(V)); CK(w.mark.reserve(n)); CK(w.list0.reserve(n)); CK(w.list1.reserve(n));
  CK(w.pool.reserve((size_t)groups * ws_pool_cap(ctx->V)));
  CK(w.ctl.reserve(groups));
  ctx->ws_groups = groups;
  return MNB_OK;
}

static int32_t ensure_dijkstra_workspace(mnb_ctx* ctx, uint32_t groups) {
  if (groups <= ctx->dws_groups) return MNB_OK;
  DijkstraBatchBuffers& w = ctx->dws;
  w = DijkstraBatchBuffers{};        // the smaller workspace goes first: batch_shape has counted its bytes as available
  ctx->dws_groups = 0; ctx->dws_marks_clean = false;
  const size_t n = (size_t)groups * ctx->V;
  CK(w.label.reserve(n)); CK(w.mark.reserve(n)); CK(w.list0.reserve(n)); CK(w.list1.reserve(n));
  CK(w.ctl.reserve(groups));
  ctx->dws_groups = groups;
  return MNB_OK;
}

// the kernels' views of the workspaces: plain structs of raw pointers, passed by value
static WaveWorkspace wave_workspace(const mnb_ctx* ctx) {
  const WaveBuffers& b = ctx->ws;
  WaveWorkspace w{};
  w.state = b.state; w.ext = b.ext; w.root = b.root; w.pool = b.pool; w.pool_cap = ws_pool_cap(ctx->V);
  w.last_eval = b.last_eval; w.dirty = b.dirty; w.skipw = b.skipw; w.chg = b.chg; w.ver = b.ver;
  w.mark = b.mark; w.list0 = b.list0; w.list1 = b.list1; w.ctl = b.ctl;
  return w;
}
static DijkstraBatchWorkspace dijkstra_workspace(const mnb_ctx* ctx) {
  const DijkstraBatchBuffers& b = ctx->dws;
  DijkstraBatchWorkspace w{};
  w.label = b.label; w.mark = b.mark; w.list0 = b.list0; w.list1 = b.list1; w.ctl = b.ctl;
  return w;
}

// Runs the body of a C-ABI entry point: std::bad_alloc (the host tables of a 50M-vertex map are tens of GB) becomes
// MNB_E_NOMEM, anything else MNB_E_STATE; a failed mnb_set_mesh frees what it had built so that later calls see an empty
// context instead of a half-built one.
template <class F>
static int32_t guarded(mnb_ctx* ctx, F body) {
  try {
    return body();
  } catch (const std::bad_alloc&) {
    if (ctx) ctx->err = "out of host memory";
    return MNB_E_NOMEM;
  } catch (const std::exception& ex) {
    if (ctx) ctx->err = ex.what();
    return MNB_E_STATE;
  } catch (...) {
    if (ctx) ctx->err = "unknown exception";
    return MNB_E_STATE;
  }
}

extern "C" {

int32_t mnb_create(int32_t device, mnb_ctx** out_ctx) {
  if (!out_ctx) return MNB_E_ARG;
  *out_ctx = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) return MNB_E_CUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return MNB_E_CUDA;
  if (prop.major != 9 || prop.minor != 0) return MNB_E_CUDA;   // sm_90a code loads on compute capability 9.0 only; no fallback path exists
  if (cudaSetDevice(device) != cudaSuccess) return MNB_E_CUDA;
  mnb_ctx* c = new mnb_ctx();
  c->device = device; c->sm_count = prop.multiProcessorCount;
  {
    int optin = 0;
#ifdef MNB_EMU_ACTIVE
    optin = 227 * 1024;         // (the interpreter has no device attributes; an H100's opt-in limit)
#else
    if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device) != cudaSuccess) { delete c; return MNB_E_CUDA; }
#endif
    const size_t room = (size_t)optin > GRID_STATIC_SMEM_ROOM ? (size_t)optin - GRID_STATIC_SMEM_ROOM : 0;
    c->grid_slots_max = (uint32_t)std::min<size_t>(room / GRID_SLOT_BYTES, GRID_SLOTS_MAX);
    c->grid_slots = std::min(GRID_SLOTS_DEFAULT, c->grid_slots_max);
    if (c->grid_slots == 0) { delete c; return MNB_E_CUDA; }
  }
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) { delete c; return MNB_E_CUDA; }
  cudaEventCreate(&c->ev0); cudaEventCreate(&c->ev1);
  c->d_next_query.reserve(1);
  if (cudaHostAlloc((void**)&c->h_cancel, sizeof(int), cudaHostAllocMapped) == cudaSuccess) {
    *c->h_cancel = 0;
    cudaHostGetDevicePointer((void**)&c->d_cancel, c->h_cancel, 0);
  }
  *out_ctx = c;
  return MNB_OK;
}

void mnb_destroy(mnb_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->h_cancel) cudaFreeHost(ctx->h_cancel);
  if (ctx->ev0) cudaEventDestroy(ctx->ev0);
  if (ctx->ev1) cudaEventDestroy(ctx->ev1);
  cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char* mnb_last_error(mnb_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
int32_t mnb_set_pointer_mode(mnb_ctx* ctx, int32_t mode) {
  if (!ctx || (mode != MNB_PTR_HOST && mode != MNB_PTR_DEVICE)) return MNB_E_ARG;
  ctx->ptr_mode = mode; return MNB_OK;
}
void* mnb_stream(mnb_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
uint32_t mnb_num_vertices(mnb_ctx* ctx) { return ctx ? ctx->V : 0; }
uint32_t mnb_num_faces(mnb_ctx* ctx) { return ctx ? ctx->F : 0; }
uint32_t mnb_num_edges(mnb_ctx* ctx) { return ctx ? ctx->E : 0; }

int32_t mnb_set_tuning(mnb_ctx* ctx, float band_delta, int32_t cluster_size, int32_t threads_per_cta) {
  if (!ctx) return MNB_E_ARG;
  if (band_delta > 0) {
    ctx->delta = band_delta; ctx->grid_delta = band_delta; ctx->dijkstra_grid_delta = band_delta; ctx->dijkstra_batch_delta = band_delta;
    ctx->delta_explicit = true;
  }
  if (cluster_size == 1 || cluster_size == 2 || cluster_size == 4 || cluster_size == 8 || cluster_size == 16) {
    ctx->cluster = cluster_size;
    ctx->batch_cluster = cluster_size > 8 ? 8 : cluster_size;
  } else if (cluster_size == -1) {
    ctx->cluster = -1;        // single plans on the whole grid (cooperative launch); batches keep their cluster size
  } else if (cluster_size != 0) return MNB_E_ARG;
  if (threads_per_cta == 128 || threads_per_cta == 256 || threads_per_cta == 512) { ctx->threads = threads_per_cta; ctx->grid_blocks_per_sm = 0; }
  else if (threads_per_cta != 0) return MNB_E_ARG;
  return MNB_OK;
}

int32_t mnb_get_stats(mnb_ctx* ctx, mnb_stats* out) {
  if (!ctx || !out) return MNB_E_ARG;
  *out = ctx->stats; return MNB_OK;
}

static int32_t impl_set_mesh(mnb_ctx* ctx, uint32_t V, uint32_t F, const float* pos, const uint32_t* faces,
                     const uint32_t* edges, uint32_t E) {
  if (!ctx || !pos || !faces || V == 0 || F == 0) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  free_mesh(ctx);
  try {
    ctx->topo.build(V, F, faces, edges, E);
  } catch (const std::exception& ex) {
    ctx->err = ex.what();
    return MNB_E_ARG;
  }
  HostTopology& T = ctx->topo;
  if (!ctx->layers_explicit) {
    // the compact seen-set of the layer walk (SharedSeen<uint16_t>) holds ids within +-32767 of the centre's: a neighbourhood
    // reaches a few edges out, so it pays when edges connect nearby ids (scan / Morton numbering); otherwise the 32-bit form
    uint32_t maxd = 0;
    for (size_t e = 0; e < (size_t)T.E; ++e) { const uint32_t a = T.edges[2 * e], b = T.edges[2 * e + 1]; maxd = std::max(maxd, a > b ? a - b : b - a); }
    ctx->layers_walk = (maxd <= 8000u) ? LAYERS_WALK_PF16 : LAYERS_WALK_PF32;
  }
  ctx->V = V; ctx->F = F; ctx->E = T.E; ctx->NC = T.cor_v1.size(); ctx->NA = T.vadj_nbr.size();
  const size_t NC = ctx->NC, NA = ctx->NA;
  CK(ctx->d_pos.reserve(3 * (size_t)V)); CK(ctx->d_faces.reserve(3 * (size_t)F)); CK(ctx->d_edges.reserve(2 * (size_t)T.E));
  CK(ctx->d_cor_ptr.reserve((size_t)V + 1)); CK(ctx->d_cor_idx.reserve(NC)); CK(ctx->d_cor_eid.reserve(NC));
  CK(ctx->d_cor_w.reserve(NC)); CK(ctx->d_cor_wd.reserve(NC));
  CK(ctx->d_adj_ptr.reserve((size_t)V + 1)); CK(ctx->d_adj_nbr.reserve(NA)); CK(ctx->d_adj_eid.reserve(NA)); CK(ctx->d_adj_nw.reserve(NA)); CK(ctx->d_ell_adj.reserve((size_t)V * ELL_W));
  CK(ctx->d_edge_dist.reserve((size_t)T.E)); CK(ctx->d_edge_w.reserve((size_t)T.E)); CK(ctx->d_cost.reserve((size_t)V));
  CK(ctx->d_invalid.reserve((size_t)V));
  CK(cudaMemcpyAsync(ctx->d_pos, pos, sizeof(float) * 3 * (size_t)V, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_faces, faces, sizeof(uint32_t) * 3 * (size_t)F, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_edges, T.edges.data(), sizeof(uint32_t) * 2 * (size_t)T.E, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_cor_ptr, T.vcor_ptr.data(), sizeof(uint32_t) * ((size_t)V + 1), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_adj_ptr, T.vadj_ptr.data(), sizeof(uint32_t) * ((size_t)V + 1), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_adj_nbr, T.vadj_nbr.data(), sizeof(uint32_t) * NA, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_adj_eid, T.vadj_eid.data(), sizeof(uint32_t) * NA, cudaMemcpyHostToDevice, ctx->stream));
  {
    std::vector<int4> idx(NC); std::vector<uint4> eid(NC);
    for (size_t k = 0; k < NC; ++k) {
      idx[k] = make_int4((int)T.cor_v1[k], (int)T.cor_v2[k], (int)T.cor_face[k], (int)T.cor_side[k]);   // .w: edge-side bits (topology.hpp)
      eid[k] = make_uint4(T.cor_ec[k], T.cor_eb[k], T.cor_ea[k], 0);
    }
    CK(cudaMemcpyAsync(ctx->d_cor_idx, idx.data(), sizeof(int4) * NC, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_cor_eid, eid.data(), sizeof(uint4) * NC, cudaMemcpyHostToDevice, ctx->stream));
    CK(ctx->d_face_cor.reserve(3 * (size_t)F));
    CK(cudaMemcpyAsync(ctx->d_face_cor, T.face_cor.data(), sizeof(uint32_t) * 3 * (size_t)F, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    // ELL rows: 8 slots per vertex (one 128-byte line), slot 0 carries the degree in .w
    const size_t NE = (size_t)V * ELL_W;
    std::vector<int4> eidx(NE, make_int4(ELL_EMPTY, ELL_EMPTY, -1, 0)); std::vector<uint4> eeid(NE, make_uint4(0, 0, 0, 0));
    for (uint32_t v = 0; v < V; ++v) {
      const uint32_t kb = T.vcor_ptr[v], ke = T.vcor_ptr[v + 1];
      for (uint32_t k = kb; k < ke && k - kb < ELL_W; ++k) { eidx[(size_t)v * ELL_W + (k - kb)] = idx[k]; eeid[(size_t)v * ELL_W + (k - kb)] = eid[k]; }
      eidx[(size_t)v * ELL_W].w = (int)(ke - kb);
    }
    CK(ctx->d_ell_idx.reserve(NE)); CK(ctx->d_ell_eid.reserve(NE)); CK(ctx->d_ell_w.reserve(NE)); CK(ctx->d_ell_wd.reserve(NE));
    CK(ctx->d_ell_geo.reserve(NE));
    CK(cudaMemcpyAsync(ctx->d_ell_idx, eidx.data(), sizeof(int4) * NE, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_ell_eid, eeid.data(), sizeof(uint4) * NE, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  // the host copies of the big per-corner arrays are no longer needed
  std::vector<uint32_t>().swap(T.cor_v1); std::vector<uint32_t>().swap(T.cor_v2); std::vector<uint32_t>().swap(T.cor_face);
  std::vector<uint32_t>().swap(T.cor_ec); std::vector<uint32_t>().swap(T.cor_eb); std::vector<uint32_t>().swap(T.cor_ea);
  std::vector<uint8_t>().swap(T.cor_side);
  std::vector<uint32_t>().swap(T.vadj_nbr); std::vector<uint32_t>().swap(T.vadj_eid); std::vector<uint32_t>().swap(T.face_edges);
  CK(ctx->d_face_normals.reserve(3 * (size_t)F)); CK(ctx->d_vertex_normals.reserve(3 * (size_t)V)); CK(ctx->d_border.reserve((size_t)V));
  CK(cudaMemcpyAsync(ctx->d_border, T.border.data(), (size_t)V, cudaMemcpyHostToDevice, ctx->stream));
  MNB_LAUNCH(k_face_normals, (F + 255) / 256, 256, 0, ctx->stream, ctx->d_pos, ctx->d_faces, F, ctx->d_face_normals);
  MNB_LAUNCH(k_vertex_normals, (V + 255) / 256, 256, 0, ctx->stream, ctx->d_cor_ptr, ctx->d_cor_idx, ctx->d_face_normals, V, ctx->d_vertex_normals);
  MNB_LAUNCH(k_edge_dist, (T.E + 255) / 256, 256, 0, ctx->stream, ctx->d_pos, ctx->d_edges, T.E, ctx->d_edge_dist);
  MNB_LAUNCH(k_gather_corner_w, (unsigned)((NC + 255) / 256), 256, 0, ctx->stream, ctx->d_cor_eid, ctx->d_edge_dist, NC, ctx->d_cor_wd);
  MNB_LAUNCH(k_gather_corner_w, (unsigned)(((size_t)V * ELL_W + 255) / 256), 256, 0, ctx->stream, ctx->d_ell_eid, ctx->d_edge_dist, (size_t)V * ELL_W, ctx->d_ell_wd);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(ctx->stream));
  return MNB_OK;
}

int32_t mnb_get_edges(mnb_ctx* ctx, uint32_t* out_edges) {
  if (!ctx || !out_edges || !ctx->V) return MNB_E_ARG;
  std::memcpy(out_edges, ctx->topo.edges.data(), sizeof(uint32_t) * 2 * (size_t)ctx->E);
  return MNB_OK;
}

int32_t mnb_get_edge_distances(mnb_ctx* ctx, float* out) {
  if (!ctx || !out || !ctx->V) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(CallerArrays(ctx).copy_out(out, ctx->d_edge_dist.p, ctx->E));
  CK(cudaStreamSynchronize(ctx->stream));
  return MNB_OK;
}

static int32_t install_weights(mnb_ctx* ctx) {
  MNB_LAUNCH(k_gather_corner_w, (unsigned)((ctx->NC + 255) / 256), 256, 0, ctx->stream, ctx->d_cor_eid, ctx->d_edge_w, ctx->NC, ctx->d_cor_w);
  MNB_LAUNCH(k_gather_corner_w, (unsigned)(((size_t)ctx->V * ELL_W + 255) / 256), 256, 0, ctx->stream, ctx->d_ell_eid, ctx->d_edge_w, (size_t)ctx->V * ELL_W, ctx->d_ell_w);
  MNB_LAUNCH(k_corner_geo, (unsigned)(((size_t)ctx->V * ELL_W + 255) / 256), 256, 0, ctx->stream, ctx->d_ell_w, (size_t)ctx->V * ELL_W, ctx->d_ell_geo);
  ctx->adj_dirty = true;        // adjacency form of the weights: only the Dijkstra planner reads it (ensure_adj_tables)
  CK(cudaGetLastError());
  // scale of the potentials: mean finite edge weight (see mnb_ctx::delta_explicit)
  CK(ctx->d_wsum.reserve(2));
  CK(cudaMemsetAsync(ctx->d_wsum, 0, 2 * sizeof(double), ctx->stream));
  MNB_LAUNCH(k_weight_scale, 2 * ctx->sm_count, 256, 0, ctx->stream, (const float*)ctx->d_edge_w, ctx->E, ctx->d_wsum);
  CK(cudaGetLastError());
  double hs[2] = {0.0, 0.0};
  CK(cudaMemcpyAsync(hs, ctx->d_wsum, sizeof(hs), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->w_mean = hs[1] > 0 ? (float)(hs[0] / hs[1]) : 0.0f;
  if (!ctx->delta_explicit && ctx->w_mean > 0) {
    // Single plans: the band should hold about as many candidates as the grid has sweep slots (SM count x GridStage slots);
    // beyond that the in-round sweeps cannot follow and the band's rows fall out of the L2.  A front is ~3 sqrt(V) vertices
    // long on a compact map and a hop is ~1.35 w deep.  5 M vertices: GRID_BAND_W for both planners; with 132 SMs and 2048
    // slots the band narrows above ~9 M vertices (24 w at 25 M).
    const float slots = (float)ctx->sm_count * (float)ctx->grid_slots;
    const float hops = slots / (3.0f * sqrtf((float)ctx->V));
    const float k = fmaxf(4.0f, 1.35f * hops);
    ctx->delta = 2.5f * ctx->w_mean;
    ctx->grid_delta = fminf(GRID_BAND_W, k) * ctx->w_mean;
    ctx->dijkstra_grid_delta = fminf(GRID_BAND_W, k) * ctx->w_mean;
    ctx->dijkstra_batch_delta = DIJKSTRA_BATCH_DELTA_W * ctx->w_mean;
  }
  ctx->costs_set = true;
  return MNB_OK;
}

// the vertex->neighbour form of the installed weights (CSR {neighbour, weight} + the 8-slot ELL rows of k_dijkstra_grid)
static int32_t ensure_adj_tables(mnb_ctx* ctx) {
  if (!ctx->adj_dirty) return MNB_OK;
  MNB_LAUNCH(k_gather_adj_w, (unsigned)((ctx->NA + 255) / 256), 256, 0, ctx->stream, ctx->d_adj_nbr, ctx->d_adj_eid, ctx->d_edge_w, ctx->NA, ctx->d_adj_nw);
  MNB_LAUNCH(k_build_ell_adj, (unsigned)(((size_t)ctx->V * ELL_W + 255) / 256), 256, 0, ctx->stream, ctx->d_adj_ptr, ctx->d_adj_nw, ctx->V, ctx->d_ell_adj);
  CK(cudaGetLastError());
  ctx->adj_dirty = false;
  return MNB_OK;
}

static int32_t impl_compute_edge_weights(mnb_ctx* ctx, const float* vertex_costs, double edge_cost_factor, float* out_w) {
  if (!ctx || !vertex_costs || !ctx->V) return MNB_E_ARG;
  ++ctx->cost_gen;
  CK(cudaSetDevice(ctx->device));
  CallerArrays io(ctx);
  CK(io.copy_in(ctx->d_cost.p, vertex_costs, ctx->V));
  MNB_LAUNCH(k_edge_weights, (ctx->E + 255) / 256, 256, 0, ctx->stream, ctx->d_cost, ctx->d_edges, ctx->d_edge_dist, edge_cost_factor, ctx->E, ctx->d_edge_w);
  CK(cudaGetLastError());
  int32_t rc = install_weights(ctx);
  if (rc != MNB_OK) return rc;
  if (out_w) CK(io.copy_out(out_w, ctx->d_edge_w.p, ctx->E));
  CK(cudaStreamSynchronize(ctx->stream));
  return MNB_OK;
}

static int32_t impl_set_costs(mnb_ctx* ctx, const float* vertex_costs, const float* edge_weights, const uint8_t* invalid) {
  if (!ctx || !vertex_costs || !edge_weights || !ctx->V) return MNB_E_ARG;
  ++ctx->cost_gen;
  CK(cudaSetDevice(ctx->device));
  CallerArrays io(ctx);
  CK(io.copy_in(ctx->d_cost.p, vertex_costs, ctx->V));
  CK(io.copy_in(ctx->d_edge_w.p, edge_weights, ctx->E));
  if (invalid) CK(io.copy_in(ctx->d_invalid.p, invalid, ctx->V));
  ctx->has_invalid = invalid != nullptr;
  int32_t rc = install_weights(ctx);
  if (rc != MNB_OK) return rc;
  CK(cudaStreamSynchronize(ctx->stream));
  return MNB_OK;
}

int32_t mnb_cancel(mnb_ctx* ctx) {
  if (!ctx || !ctx->h_cancel) return MNB_E_ARG;
  *(volatile int*)ctx->h_cancel = 1;
  return MNB_OK;
}

}  // extern "C"


static RepulsiveField repulsive_field_of(mnb_ctx* ctx) {
  RepulsiveField L{};
  L.dist = ctx->d_infl_dist; L.vec = ctx->d_infl_vec;
  L.inscribed_radius = ctx->infl_params.inscribed_radius; L.inflation_radius = ctx->infl_params.inflation_radius;
  L.inscribed_radius_f = (float)ctx->infl_params.inscribed_radius;
  L.lethal_value = (float)ctx->infl_params.lethal_value; L.inscribed_value = (float)ctx->infl_params.inscribed_value;
  return L;
}

extern "C" {

// The repulsive field from the labels of the last inflation wave in the workspace (the wave ran with the invalid mask
// d_infl_invalid if infl_had_invalid): of every vertex (list null), or of the vertices of a list whose clusters that
// wave labelled (mnb_inflation_repair) -- the vectors of a cluster depend on sources in that cluster only.
static int32_t infl_vector_field(mnb_ctx* ctx, const uint32_t* list, uint32_t n, unsigned& launches) {
  const size_t V = ctx->V;
  CK(ctx->d_infl_vec.reserve(3 * V)); CK(ctx->d_infl_src.reserve(V)); CK(ctx->d_infl_flag.reserve(2));
  InflVecArgs a{};
  a.V = ctx->V; a.pos = ctx->d_pos; a.faces = ctx->d_faces; a.cor_ptr = ctx->d_cor_ptr; a.cor_idx = ctx->d_cor_idx; a.cor_wd = ctx->d_cor_wd;
  a.cor_eid = ctx->d_cor_eid; a.adj_ptr = ctx->d_adj_ptr; a.adj_nbr = ctx->d_adj_nbr; a.invalid = ctx->infl_had_invalid ? ctx->d_infl_invalid.p : nullptr; a.ws = wave_workspace(ctx);
  a.max_distance = (float)ctx->infl_params.inflation_radius; a.vec = ctx->d_infl_vec; a.src = ctx->d_infl_src; a.flag = ctx->d_infl_flag;
  CK(cudaMemsetAsync(ctx->d_infl_flag, 0, 2 * sizeof(unsigned int), ctx->stream));
  if (list) {
    MNB_LAUNCH(k_infl_vec_lethal_list, (n + 127) / 128, 128, 0, ctx->stream, a, list, n);
    MNB_LAUNCH(k_infl_vec_sources_list, (n + 127) / 128, 128, 0, ctx->stream, a, list, n);
  } else {
    MNB_LAUNCH(k_infl_vec_lethal, (ctx->V + 127) / 128, 128, 0, ctx->stream, a);
    MNB_LAUNCH(k_infl_vec_sources, (ctx->V + 127) / 128, 128, 0, ctx->stream, a);
  }
  CK(cudaGetLastError());
  launches += 2;
  // fixed point over the acyclic source relation: its depth is bounded by the number of rounds the wave took
  const unsigned max_sweeps = (unsigned)ctx->infl_rounds + 8u;
  unsigned int flag[2] = {1u, 0u};
  for (unsigned it = 0; it < max_sweeps && flag[0]; ++it, ++launches) {
    CK(cudaMemsetAsync(ctx->d_infl_flag, 0, sizeof(unsigned int), ctx->stream));
    if (list) MNB_LAUNCH(k_infl_vec_sweep_list, (n + 255) / 256, 256, 0, ctx->stream, a, list, n);
    else MNB_LAUNCH(k_infl_vec_sweep, (ctx->V + 255) / 256, 256, 0, ctx->stream, a);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(flag, ctx->d_infl_flag, sizeof(flag), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  if (flag[1]) { ctx->err = "inflation vector field: a vertex has more than 24 faces with two lethal vertices"; return MNB_E_NOMEM; }
  if (flag[0]) { ctx->err = "inflation vector field did not reach its fixed point"; return MNB_E_STATE; }
  return MNB_OK;
}

static int32_t impl_inflation_vector_map(mnb_ctx* ctx, float* out_vectors) {
  if (!ctx || !ctx->V) return MNB_E_ARG;
  if (ctx->infl_field_resident) {            // kept up to date by mnb_inflation_repair: no labels needed
    CK(cudaSetDevice(ctx->device));
    if (out_vectors) CK(CallerArrays(ctx).copy_out(out_vectors, ctx->d_infl_vec.p, 3 * (size_t)ctx->V));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->stats = mnb_stats{};
    return MNB_OK;
  }
  if (!ctx->infl_labels_valid) {
    ctx->err = "mnb_inflation_vector_map needs the labels of the last mnb_inflate / mnb_inflation_update: call it before the next planner call on this context";
    return MNB_E_STATE;
  }
  CK(cudaSetDevice(ctx->device));
  const size_t V = ctx->V;
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  unsigned launches = 0;
  const int32_t rc = infl_vector_field(ctx, nullptr, 0, launches);
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  if (rc != MNB_OK) return rc;
  if (out_vectors) CK(CallerArrays(ctx).copy_out(out_vectors, ctx->d_infl_vec.p, 3 * V));
  CK(cudaStreamSynchronize(ctx->stream));
  simple_stats(ctx, launches, ctx->V);
  ctx->stats.rounds = ctx->infl_rounds;
  ctx->infl_field_valid = true;
  return MNB_OK;
}

int32_t mnb_set_repulsive_field(mnb_ctx* ctx, int32_t enable) {
  if (!ctx) return MNB_E_ARG;
  if (enable && !ctx->infl_field_valid) { ctx->err = "mnb_set_repulsive_field needs mnb_inflation_vector_map first"; return MNB_E_STATE; }
  ctx->repulsive_on = enable != 0;
  return MNB_OK;
}

static int32_t impl_inflation_vector_at(mnb_ctx* ctx, uint32_t n, const uint32_t* faces_q, const float* bary, float* out) {
  if (!ctx || !ctx->V || !faces_q || !bary || !out || n == 0) return MNB_E_ARG;
  if (!ctx->infl_field_valid) { ctx->err = "mnb_inflation_vector_at needs mnb_inflation_vector_map first"; return MNB_E_STATE; }
  for (uint32_t i = 0; ctx->ptr_mode == MNB_PTR_HOST && i < n; ++i) if (faces_q[i] >= ctx->F) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  CallerArrays io(ctx);
  DeviceBuffer<uint32_t> d_f; DeviceBuffer<float> d_b, d_o;      // host-pointer mode: device copies for this call
  const uint32_t* const f = io.in(faces_q, d_f, n);
  const float* const b = io.in(bary, d_b, 3 * (size_t)n);
  float* const o = io.out(out, d_o, 3 * (size_t)n);
  CK(io.status());
  MNB_LAUNCH(k_inflation_vector_at, (n + 127) / 128, 128, 0, ctx->stream, repulsive_field_of(ctx), (const uint32_t*)ctx->d_faces, n, f, b, o);
  CK(cudaGetLastError());
  CK(io.copy_back());
  CK(cudaStreamSynchronize(ctx->stream));
  return MNB_OK;
}

}  // extern "C"

template <class KArgs>
static cudaError_t launch_cluster(void (*kern)(const KArgs), const KArgs& args, int cs, unsigned blocks, int threads,
                                  cudaStream_t stream) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = 0; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = cs > 1 ? 1 : 0;
  if (cs > 8) {
    cudaError_t e = cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e != cudaSuccess) return e;
  }
  return cudaLaunchKernelEx(&cfg, kern, args);
}

// cooperative (grid-synchronising) launch of a kernel that takes one argument struct
template <class KArgs>
static cudaError_t launch_cooperative(void (*kern)(const KArgs), const KArgs& args, unsigned blocks, int threads, cudaStream_t stream,
                                      size_t smem = 0) {
#ifdef MNB_EMU_ACTIVE
  (void)stream;
  return emu::launch(kern, blocks, (unsigned)threads, smem, 1u, true, args);
#else
  void* kargs[] = {(void*)&args};
  return cudaLaunchCooperativeKernel((const void*)kern, dim3(blocks), dim3(threads), kargs, smem, stream);
#endif
}

// A whole-grid kernel (index k of mnb_ctx::grid_smem_set) with the dynamic shared memory of ctx->grid_slots GridStage slots:
// allows that much, and checks that one CTA of `threads` still fits on an SM (the cooperative launch needs every CTA resident).
template <class KArgs>
static cudaError_t grid_kernel_smem(mnb_ctx* ctx, void (*kern)(const KArgs), int k, int threads, size_t& smem) {
  smem = (size_t)ctx->grid_slots * GRID_SLOT_BYTES;
  if (ctx->grid_smem_set[k] == smem) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int nb = 0;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, threads, smem)) != cudaSuccess) return e;
  if (nb < 1) return cudaErrorInvalidValue;        // (no CTA fits)
  ctx->grid_smem_set[k] = smem;
  return cudaSuccess;
}

// free and total device memory (sizes the workspaces that are capped by memory)
static cudaError_t device_memory(int device, size_t* free_b, size_t* total_b) {
#ifdef MNB_EMU_ACTIVE
  // the CPU interpreter of the kernels (tests/emu) models no memory budget: its whole arena counts as free
  cudaDeviceProp prop;
  const cudaError_t e = cudaGetDeviceProperties(&prop, device);
  *free_b = prop.totalGlobalMem; *total_b = prop.totalGlobalMem;
  return e;
#else
  (void)device;
  return cudaMemGetInfo(free_b, total_b);
#endif
}

// Calls launch(std::integral_constant<int, CS>()) with the cluster size cs as a compile-time constant: 1, 2, 4 and 8 as
// given, anything else as MAX_CS (8 for the batch kernels, 16 for single plans), so a kernel template is instantiated for
// exactly these sizes.
template <int MAX_CS, class F>
static cudaError_t with_cluster_size(int cs, F&& launch) {
  switch (cs) {
    case 1: return launch(std::integral_constant<int, 1>());
    case 2: return launch(std::integral_constant<int, 2>());
    case 4: return launch(std::integral_constant<int, 4>());
    case 8: return launch(std::integral_constant<int, 8>());
    default: return launch(std::integral_constant<int, MAX_CS>());
  }
}

// Launch shape of a batch of n wavefronts on kernel `kern` (its one-CTA instantiation).  Concurrent wavefronts: the CTA
// slots its occupancy allows (at most MNB_BATCH_MINBLOCKS per SM), capped by the device memory a workspace of per_group
// bytes per wavefront may take -- the free memory plus the `current` groups a larger workspace would replace, less a
// reserve (512 MB or 1/32 of the device); MNB_E_NOMEM if not even one fits.  CTAs per wavefront (unless mnb_set_tuning
// fixed them): one when the wavefronts fill the machine, a cluster when there are fewer of them than CTA slots, so that
// the SMs do not idle (strong scaling across GPUs hands every rank a fraction of the batch).
template <class KArgs>
static int32_t batch_shape(mnb_ctx* ctx, void (*kern)(const KArgs), uint32_t n, size_t per_group, uint32_t current,
                           const char* what, int* cs_out, unsigned* groups_out) {
  int per_sm = 1;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, MNB_BATCH_THREADS, 0));
  const unsigned slots = (unsigned)(ctx->sm_count * std::max(1, std::min(per_sm, (int)MNB_BATCH_MINBLOCKS)));
  size_t free_b = 0, total_b = 0;
  CK(device_memory(ctx->device, &free_b, &total_b));
  const size_t avail = free_b + (size_t)current * per_group;
  const size_t reserve = std::max<size_t>((size_t)512 << 20, total_b / 32);
  const size_t mem_groups = avail > reserve ? (avail - reserve) / per_group : 0;
  if (mem_groups == 0) { ctx->err = std::string("not enough free device memory for one ") + what + " wavefront"; return MNB_E_NOMEM; }
  const unsigned want = (unsigned)std::min<size_t>(std::min<size_t>(n, slots), mem_groups);
  int cs = ctx->batch_cluster;
  if (cs <= 0) { cs = 1; while (cs < 8 && (unsigned)(2 * cs) * want <= slots) cs *= 2; }
  *cs_out = cs;
  *groups_out = std::min(want, std::max(1u, slots / (unsigned)cs));
  return MNB_OK;
}

// One batch of n waves (mnb_cvp_batch_fields, mnb_dijkstra_batch): kernel(std::integral_constant<int, CS>()) is the
// kernel at cluster size CS.  Its one-CTA form sizes the launch (batch_shape), prepare(groups) grows the workspace and
// fills args, and the launch at the chosen cluster size is timed by ev0 / ev1.
template <class Kernel, class KArgs, class Prepare>
static int32_t run_batch(mnb_ctx* ctx, Kernel kernel, const KArgs& args, uint32_t n, size_t per_group, uint32_t current,
                         const char* what, Prepare prepare, unsigned* groups_out) {
  int cs = 1; unsigned groups = 1;
  int32_t rc = batch_shape(ctx, kernel(std::integral_constant<int, 1>()), n, per_group, current, what, &cs, &groups);
  if (rc != MNB_OK || (rc = prepare(groups)) != MNB_OK) return rc;
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  const unsigned blocks = groups * (unsigned)cs;
  const cudaError_t e = with_cluster_size<8>(cs, [&](auto c) {
    return launch_cluster(kernel(c), args, decltype(c)::value, blocks, MNB_BATCH_THREADS, ctx->stream);
  });
  if (e != cudaSuccess) { ctx->err = std::string(what) + " batch launch: " + cudaGetErrorString(e); return MNB_E_CUDA; }
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  *groups_out = groups;
  return MNB_OK;
}

static int32_t finish_stats(mnb_ctx* ctx, unsigned groups, unsigned launches, const GroupCtl* ctl = nullptr) {
  std::vector<GroupCtl> h(groups);
  CK(cudaMemcpyAsync(h.data(), ctl ? ctl : ctx->ws.ctl, sizeof(GroupCtl) * groups, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->stats.rounds = 0; ctx->stats.recomputes = 0; ctx->stats.settled = 0;
  ctx->stats.skipped = 0; ctx->stats.deep_labels = 0; ctx->stats.pool_words = 0;
  for (auto& c : h) { ctx->stats.deep_labels += c.deep_labels; ctx->stats.pool_words = std::max<uint64_t>(ctx->stats.pool_words, c.pool_top); }
  for (auto& c : h) { ctx->stats.rounds += c.rounds; ctx->stats.recomputes += c.recomputes; ctx->stats.settled += c.settled; ctx->stats.skipped += c.skipped; }
  ctx->stats.kernel_launches = launches;
  float ms = 0; cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1); ctx->stats.kernel_ms = ms;
  if (getenv("MNB_PHASE_TIMING")) for (auto& c : h) fprintf(stderr, "[mnb] rounds %llu: CTA0 cycles work %llu flush %llu sync %llu (per round %.0f / %.0f / %.0f) main-pass cycles %llu candidates %llu (queued for 8 lanes %llu) | sweeps: dirty %llu polled %llu poll-cycles %llu eval-cycles %llu | main pass, one-thread phase cycles %llu\n", c.rounds, c.t_work, c.t_flush, c.t_sync, (double)c.t_work / (double)(c.rounds ? c.rounds : 1), (double)c.t_flush / (double)(c.rounds ? c.rounds : 1), (double)c.t_sync / (double)(c.rounds ? c.rounds : 1), c.t_ph[0], c.t_ph[2], c.t_ph[1], c.t_ph[3], c.t_ph[4], c.t_ph[5], c.t_ph[6], c.t_ph[7]);
  for (auto& c : h)
    if (c.watchdog) { ctx->err = "wavefront did not converge within the round watchdog"; return MNB_E_STATE; }
  for (auto& c : h)
    if (c.pool_overflow) { ctx->err = "level pool exhausted: the cascades of this map nest deeper than the workspace holds (result discarded)"; return MNB_E_NOMEM; }
  return MNB_OK;
}

static int32_t ensure_out(mnb_ctx* ctx, size_t n_dist, bool aux) {
  CK(ctx->d_out_dist.reserve(n_dist));
  if (aux) { CK(ctx->d_out_pred.reserve(ctx->V)); CK(ctx->d_out_dir.reserve(ctx->V)); CK(ctx->d_out_cut.reserve(ctx->V)); }
  return MNB_OK;
}

static int32_t ensure_seeds(mnb_ctx* ctx, uint32_t n) {
  CK(ctx->d_seed_faces.reserve(n)); CK(ctx->d_seed_pos.reserve(3 * (size_t)n));
  return MNB_OK;
}

// The targets of a cost-matrix call (mnb_dijkstra_matrix, mnb_cvp_matrix): host list, [n][m] output in the pointer mode.
struct MatrixRequest { uint32_t m; const uint32_t* targets; float* out; };

// MNB_INVALID_GOAL if a target is >= V (nothing written)
static int32_t check_targets(mnb_ctx* ctx, const MatrixRequest* mx) {
  if (mx) for (uint32_t j = 0; j < mx->m; ++j) if (mx->targets[j] >= ctx->V) return MNB_INVALID_GOAL;
  return MNB_OK;
}

// Uploads the target list and the bitmap of the distinct targets (ctx buffers, freed with the mesh) and fills tg but out.
static int32_t upload_targets(mnb_ctx* ctx, const MatrixRequest& mx, TargetSet& tg) {
  const size_t words = ((size_t)ctx->V >> 5) + 1;
  CK(ctx->d_target_bits.reserve(words)); CK(ctx->d_targets.reserve(mx.m));
  std::vector<uint32_t> bits(words, 0u);     // (a copy from pageable memory has read it when cudaMemcpyAsync returns)
  uint32_t distinct = 0;
  for (uint32_t j = 0; j < mx.m; ++j) {
    const uint32_t v = mx.targets[j], bit = 1u << (v & 31);
    if (!(bits[v >> 5] & bit)) { bits[v >> 5] |= bit; ++distinct; }
  }
  CK(cudaMemcpyAsync(ctx->d_target_bits, bits.data(), sizeof(uint32_t) * words, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_targets, mx.targets, sizeof(uint32_t) * mx.m, cudaMemcpyHostToDevice, ctx->stream));
  tg.list = ctx->d_targets; tg.bits = ctx->d_target_bits; tg.m = mx.m; tg.distinct = distinct;
  return MNB_OK;
}

// The changed vertices of a field repair (mnb_dijkstra_batch_repair): host list, any order, duplicates allowed.
struct RepairRequest { uint32_t n; const uint32_t* changed; };

// MNB_E_ARG if a changed vertex is >= V (nothing written)
static int32_t check_changed(mnb_ctx* ctx, const RepairRequest* rq) {
  if (rq) for (uint32_t i = 0; i < rq->n; ++i) if (rq->changed[i] >= ctx->V) return MNB_E_ARG;
  return MNB_OK;
}

// Uploads the distinct changed vertices and their bitmap (ctx buffers, freed with the mesh), clears the log lengths of the
// groups and fills cs.
static int32_t upload_changed(mnb_ctx* ctx, const RepairRequest& rq, unsigned groups, RepairSet& cs) {
  const size_t words = ((size_t)ctx->V >> 5) + 1;
  std::vector<uint32_t> bits(words, 0u), list;     // (a copy from pageable memory has read it when cudaMemcpyAsync returns)
  list.reserve(rq.n);
  for (uint32_t i = 0; i < rq.n; ++i) {
    const uint32_t v = rq.changed[i], bit = 1u << (v & 31);
    if (!(bits[v >> 5] & bit)) { bits[v >> 5] |= bit; list.push_back(v); }
  }
  CK(ctx->d_repair_bits.reserve(words)); CK(ctx->d_repair_chg.reserve(list.size())); CK(ctx->d_repair_log_n.reserve(groups));
  CK(cudaMemcpyAsync(ctx->d_repair_bits, bits.data(), sizeof(uint32_t) * words, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_repair_chg, list.data(), sizeof(uint32_t) * list.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(ctx->d_repair_log_n, 0, sizeof(unsigned int) * groups, ctx->stream));
  cs.list = ctx->d_repair_chg; cs.bits = ctx->d_repair_bits; cs.n = (uint32_t)list.size(); cs.log_n = ctx->d_repair_log_n;
  return MNB_OK;
}

static void fill_cvp_args(mnb_ctx* ctx, CvpKernelArgs& a) {
  a.V = ctx->V; a.pos = ctx->d_pos; a.faces = ctx->d_faces; a.cor_ptr = ctx->d_cor_ptr; a.cor_idx = ctx->d_cor_idx;
  a.cor_w = ctx->d_cor_w; a.ell_idx = ctx->d_ell_idx; a.ell_w = ctx->d_ell_w; a.ell_geo = ctx->d_ell_geo; a.cost = ctx->d_cost; a.invalid = ctx->has_invalid ? ctx->d_invalid.p : nullptr; a.ws = wave_workspace(ctx);
  a.seed_faces = ctx->d_seed_faces; a.seed_pos = ctx->d_seed_pos; a.delta = ctx->delta; a.next_query = ctx->d_next_query;
  a.cancel_flag = ctx->d_cancel; a.max_rounds = watchdog_rounds(ctx->V); a.sweeps = 0;
  a.hop = ctx->w_mean > 0 ? 1.35f * ctx->w_mean : 0.16f;
}

// A single plan's wave on the workspace of a.ws: k_cvp_grid or, with mnb_set_tuning(cluster >= 1), k_cvp<CS> -- in the
// resumed form with RESUME (mnb_cvp_replan) -- then the epilogue (k_cvp_epilogue, k_cvp_epilogue_csr).
constexpr unsigned SINGLE_CVP_LAUNCHES = 3;
template <bool RESUME>
static int32_t launch_single_cvp(mnb_ctx* ctx, CvpKernelArgs a) {
  if (ctx->cluster == -1) {
    a.delta = ctx->grid_delta;
    a.slots = ctx->grid_slots;
    size_t smem = 0;
    CK(grid_kernel_smem(ctx, k_cvp_grid<RESUME>, RESUME ? 1 : 0, ctx->threads, smem));
    if (ctx->grid_blocks_per_sm == 0) {
      int nb = 0;
      CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_cvp_grid<RESUME>, ctx->threads, smem));
      ctx->grid_blocks_per_sm = nb > MNB_GRID_MINBLOCKS ? MNB_GRID_MINBLOCKS : nb;
      if (nb <= 0) { ctx->err = "k_cvp_grid cannot be resident"; return MNB_E_CUDA; }
    }
    CK(launch_cooperative(k_cvp_grid<RESUME>, a, (unsigned)(ctx->sm_count * ctx->grid_blocks_per_sm), ctx->threads, ctx->stream, smem));
  } else {
    const cudaError_t e = with_cluster_size<16>(ctx->cluster, [&](auto c) {
      constexpr int CS = decltype(c)::value;
      return launch_cluster(k_cvp<CS, RESUME>, a, CS, (unsigned)CS, MNB_CVP_THREADS, ctx->stream);
    });
    if (e != cudaSuccess) { ctx->err = std::string("cvp launch: ") + cudaGetErrorString(e); return MNB_E_CUDA; }
  }
  CK(cudaMemsetAsync(&a.ws.ctl->epi_csr, 0, sizeof(unsigned int), ctx->stream));
  const unsigned epi_blocks = (ctx->V + MNB_EPILOGUE_THREADS - 1) / MNB_EPILOGUE_THREADS;
  if (ctx->cvp_epilogue == 1) MNB_LAUNCH(k_cvp_epilogue<true>, epi_blocks, MNB_EPILOGUE_THREADS, 0, ctx->stream, a, a.ws.ctl);
  else MNB_LAUNCH(k_cvp_epilogue<false>, epi_blocks, MNB_EPILOGUE_THREADS, 0, ctx->stream, a, a.ws.ctl);
  ctx->epi_in_rw = a.ws.ctl == ctx->rw.ctl.p;
  MNB_LAUNCH(k_cvp_epilogue_csr, (unsigned)(4 * ctx->sm_count), 256, 0, ctx->stream, a, a.ws.ctl);   // (grid-stride over the list)
  CK(cudaGetLastError());
  return MNB_OK;
}

// After the launches of a single plan: the copies back, the stats and the outcome (cvp:888-918); a plan that is not
// cancelled becomes the last plan (mnb_cvp_backtrack, mnb_vector_map).
static int32_t single_cvp_outcome(mnb_ctx* ctx, const CvpKernelArgs& a, CallerArrays& io, uint32_t seed_face, const float seed_pos[3],
                                  int64_t robot_face, unsigned launches) {
  int32_t rc;
  CK(io.copy_back());
  uint32_t rf[3] = {0, 0, 0}, rp[3] = {0, 0, 0};
  if (robot_face >= 0) {
    CK(cudaMemcpyAsync(rf, ctx->d_faces + 3 * (size_t)robot_face, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < 3; ++k)
      CK(cudaMemcpyAsync(&rp[k], a.out_pred + rf[k], sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  }
  ctx->last_valid = false;
  if ((rc = finish_stats(ctx, 1, launches, a.ws.ctl)) != MNB_OK) return rc;
  if (ctx->h_cancel && *ctx->h_cancel) return MNB_CANCELED;
  ctx->last_pred = a.out_pred; ctx->last_dir = a.out_dir; ctx->last_cut = a.out_cut; ctx->last_seed_face = seed_face;
  for (int k = 0; k < 3; ++k) ctx->last_seed_pos[k] = seed_pos[k];
  ctx->last_valid = true;
  if (robot_face >= 0) {
    bool any = false;
    for (int k = 0; k < 3; ++k) if (rp[k] != rf[k]) any = true;
    if (!any && (uint32_t)robot_face != seed_face) return MNB_NO_PATH_FOUND;
  }
  return MNB_SUCCESS;
}

extern "C" {

static int32_t impl_cvp(mnb_ctx* ctx, uint32_t seed_face, const float seed_pos[3], int64_t robot_face, double cost_limit,
                double goal_dist_offset, float* out_dist, uint32_t* out_pred, float* out_direction, int32_t* out_cut) {
  if (!ctx || !seed_pos || !ctx->V) return MNB_E_ARG;
  if (!ctx->costs_set) { ctx->err = "mnb_set_costs / mnb_compute_edge_weights not called"; return MNB_E_STATE; }
  if (seed_face >= ctx->F) return MNB_INVALID_START;
  if (robot_face >= (int64_t)ctx->F) return MNB_INVALID_GOAL;
  CK(cudaSetDevice(ctx->device));
  int32_t rc;
  if ((rc = ensure_workspace(ctx, 1)) != MNB_OK) return rc;
  if ((rc = ensure_seeds(ctx, 1)) != MNB_OK) return rc;
  // every row is produced without the caller's array too: the outcome code and mnb_cvp_backtrack read them
  CallerArrays io(ctx);
  if ((rc = ensure_out(ctx, (io.device() && out_dist) ? 0 : (size_t)ctx->V, true)) != MNB_OK) return rc;
  float* const o_dist = io.needed(out_dist, ctx->d_out_dist.p, ctx->V);
  uint32_t* const o_pred = io.needed(out_pred, ctx->d_out_pred.p, ctx->V);
  float* const o_dir = io.needed(out_direction, ctx->d_out_dir.p, ctx->V);
  int32_t* const o_cut = io.needed(out_cut, ctx->d_out_cut.p, ctx->V);
  if (ctx->h_cancel) *ctx->h_cancel = 0;     // cvp:679 "reset cancel planning"
  ctx->infl_labels_valid = false;            // the wavefront workspace is shared with the inflation wave
  CK(cudaMemcpyAsync(ctx->d_seed_faces, &seed_face, sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_seed_pos, seed_pos, 3 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(ctx->ws.ctl, 0, sizeof(GroupCtl), ctx->stream));
  CvpKernelArgs a{};
  fill_cvp_args(ctx, a);
  a.n_queries = 1; a.robot_face = robot_face; a.cost_limit = cost_limit; a.goal_dist_offset = goal_dist_offset;
  a.sweeps = ctx->sweeps;
  a.out_dist = o_dist; a.out_pred = o_pred; a.out_dir = o_dir; a.out_cut = o_cut;
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  if ((rc = launch_single_cvp<false>(ctx, a)) != MNB_OK) return rc;
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  return single_cvp_outcome(ctx, a, io, seed_face, seed_pos, robot_face, SINGLE_CVP_LAUNCHES);
}

// mnb_cvp_replan: the arguments of mnb_cvp plus the union of the changed sets of the mnb_update_vertex_costs calls since
// the resident wave.  The result is mnb_cvp's; the wave runs in the resident workspace and resumes from T0 when the last
// successful replan had the same seed face, seed position and cost limit and only mnb_update_vertex_costs changed the
// costs since (DESIGN §4, "Replan").  Otherwise, or when T0 is not after every seed's pop, or the level pool is more than
// half full, or the resumed wave would overflow it, the call runs one whole wave there.
static int32_t impl_cvp_replan(mnb_ctx* ctx, uint32_t seed_face, const float seed_pos[3], int64_t robot_face, double cost_limit,
                               double goal_dist_offset, uint32_t n_changed, const uint32_t* changed,
                               float* out_dist, uint32_t* out_pred, float* out_direction, int32_t* out_cut) {
  if (!ctx || !seed_pos || !ctx->V || (n_changed && !changed)) return MNB_E_ARG;
  const RepairRequest rq{n_changed, changed};
  int32_t rc;
  if ((rc = check_changed(ctx, &rq)) != MNB_OK) return rc;
  if (!ctx->costs_set) { ctx->err = "mnb_set_costs / mnb_compute_edge_weights not called"; return MNB_E_STATE; }
  if (seed_face >= ctx->F) return MNB_INVALID_START;
  if (robot_face >= (int64_t)ctx->F) return MNB_INVALID_GOAL;
  CK(cudaSetDevice(ctx->device));
  const size_t V = ctx->V;
  WaveBuffers& w = ctx->rw;
  CK(w.state.reserve(V)); CK(w.ext.reserve(V)); CK(w.root.reserve(V)); CK(w.chg.reserve(V)); CK(w.ver.reserve(V));
  CK(w.mark.reserve(V)); CK(w.list0.reserve(V)); CK(w.list1.reserve(V)); CK(w.pool.reserve(ws_pool_cap(ctx->V))); CK(w.ctl.reserve(1));
  if ((rc = ensure_seeds(ctx, 1)) != MNB_OK) return rc;
  CallerArrays io(ctx);
  if ((rc = ensure_out(ctx, (io.device() && out_dist) ? 0 : V, true)) != MNB_OK) return rc;
  float* const o_dist = io.needed(out_dist, ctx->d_out_dist.p, ctx->V);
  uint32_t* const o_pred = io.needed(out_pred, ctx->d_out_pred.p, ctx->V);
  float* const o_dir = io.needed(out_direction, ctx->d_out_dir.p, ctx->V);
  int32_t* const o_cut = io.needed(out_cut, ctx->d_out_cut.p, ctx->V);
  if (ctx->h_cancel) *ctx->h_cancel = 0;
  CK(cudaMemcpyAsync(ctx->d_seed_faces, &seed_face, sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_seed_pos, seed_pos, 3 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  CvpKernelArgs a{};
  fill_cvp_args(ctx, a);
  a.ws = WaveWorkspace{};
  a.ws.state = w.state; a.ws.ext = w.ext; a.ws.root = w.root; a.ws.pool = w.pool; a.ws.pool_cap = ws_pool_cap(ctx->V);
  a.ws.chg = w.chg; a.ws.ver = w.ver; a.ws.mark = w.mark; a.ws.list0 = w.list0; a.ws.list1 = w.list1; a.ws.ctl = w.ctl;
  a.n_queries = 1; a.robot_face = robot_face; a.cost_limit = cost_limit; a.goal_dist_offset = goal_dist_offset;
  a.sweeps = ctx->sweeps;
  a.out_dist = o_dist; a.out_pred = o_pred; a.out_dir = o_dir; a.out_cut = o_cut;
  uint32_t pos_bits[3]; uint64_t limit_bits;
  std::memcpy(pos_bits, seed_pos, sizeof(pos_bits)); std::memcpy(&limit_bits, &cost_limit, sizeof(limit_bits));
  bool resume = ctx->rw_valid && ctx->rw_seed_face == seed_face && std::equal(pos_bits, pos_bits + 3, ctx->rw_seed_pos) &&
                ctx->rw_cost_limit == limit_bits && ctx->rw_cost_gen == ctx->cost_gen && ctx->rw_pool_top <= ws_pool_cap(ctx->V) / 2;
  ctx->rw_valid = false;                       // until this call has succeeded
  unsigned launches = 0;
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  if (resume) {
    const unsigned blocks = std::max(1u, std::min((n_changed + 255u) / 256u, 2u * (unsigned)ctx->sm_count));
    CK(ctx->d_replan_chg.reserve(std::max(1u, n_changed))); CK(ctx->d_replan_t0.reserve(REPLAN_T0_WORDS + 6 * (size_t)blocks));
    if (n_changed) CK(cudaMemcpyAsync(ctx->d_replan_chg, changed, sizeof(uint32_t) * n_changed, cudaMemcpyHostToDevice, ctx->stream));
    ReplanArgs r{};
    r.V = ctx->V; r.faces = ctx->d_faces; r.cor_ptr = ctx->d_cor_ptr; r.cor_idx = ctx->d_cor_idx; r.cost = ctx->d_cost;
    r.invalid = a.invalid; r.cost_limit = cost_limit; r.ws = a.ws; r.changed = ctx->d_replan_chg; r.n_changed = n_changed;
    r.seed_face = seed_face; r.robot_face = robot_face; r.t0 = ctx->d_replan_t0;
    MNB_LAUNCH(k_replan_t0, blocks, 256, 0, ctx->stream, r);
    MNB_LAUNCH(k_replan_t0_final, 1, 256, 0, ctx->stream, r, blocks);
    CK(cudaGetLastError());
    launches += 2;
    uint32_t ok = 0;
    CK(cudaMemcpyAsync(&ok, ctx->d_replan_t0.p + 6, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    resume = ok != 0;
    if (resume) {
      const unsigned vb = (unsigned)((V + 255) / 256);
      MNB_LAUNCH(k_replan_rollback, vb, 256, 0, ctx->stream, r);
      MNB_LAUNCH(k_replan_frontier, vb, 256, 0, ctx->stream, r);
      CK(cudaGetLastError());
      CvpKernelArgs ra = a;
      if (ctx->replan_pool_room) ra.ws.pool_cap = std::min<uint32_t>(ra.ws.pool_cap, ctx->rw_pool_top + ctx->replan_pool_room);
      if ((rc = launch_single_cvp<true>(ctx, ra)) != MNB_OK) return rc;
      launches += 2 + SINGLE_CVP_LAUNCHES;
      // the resumed wave allocates behind the old records: if the pool ran out, the whole wave starts from an empty one
      unsigned int overflow = 0;
      CK(cudaMemcpyAsync(&overflow, &a.ws.ctl->pool_overflow, sizeof(overflow), cudaMemcpyDeviceToHost, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
      resume = overflow == 0;
    }
  }
  if (!resume) {
    CK(cudaMemsetAsync(a.ws.ctl, 0, sizeof(GroupCtl), ctx->stream));
    if ((rc = launch_single_cvp<false>(ctx, a)) != MNB_OK) return rc;
    launches += SINGLE_CVP_LAUNCHES;
  }
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  rc = single_cvp_outcome(ctx, a, io, seed_face, seed_pos, robot_face, launches);
  if (rc == MNB_SUCCESS || rc == MNB_NO_PATH_FOUND) {
    ctx->rw_valid = true; ctx->rw_seed_face = seed_face; std::copy(pos_bits, pos_bits + 3, ctx->rw_seed_pos);
    ctx->rw_cost_limit = limit_bits; ctx->rw_cost_gen = ctx->cost_gen; ctx->rw_pool_top = (uint32_t)ctx->stats.pool_words;
  }
  return rc;
}


// n full-field CVP plans in one launch, mnb_cvp_batch and mnb_cvp_batch_fields.  With vector-field outputs
// (k_cvp_batch<CS, true>) each wavefront runs the epilogue of its goal before its group takes the next one; potentials
// alone run the potentials-only kernel.  The waves share the wavefront workspace with single plans and inflation (not the
// single plan's outputs), and their number is capped by the free device memory as well as by the CTA slots.
// With mx (mnb_cvp_matrix; no row outputs) the waves run the matrix form k_cvp_batch<CS, false, CvpMatrixArgs> into mx->out.
static int32_t impl_cvp_batch_fields(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_faces, const float* seed_pos, double cost_limit,
                                     float* out_dist, uint32_t* out_pred, float* out_dir, int32_t* out_cut,
                                     const MatrixRequest* mx = nullptr) {
  if (!ctx || !seed_faces || !seed_pos || (!out_dist && !out_pred && !out_dir && !out_cut && !mx) || !ctx->V || n == 0) return MNB_E_ARG;
  if (!ctx->costs_set) { ctx->err = "costs not set"; return MNB_E_STATE; }
  for (uint32_t i = 0; i < n; ++i) if (seed_faces[i] >= ctx->F) return MNB_INVALID_START;
  int32_t rc;
  if ((rc = check_targets(ctx, mx)) != MNB_OK) return rc;
  CK(cudaSetDevice(ctx->device));
  const size_t rows = (size_t)n * ctx->V;
  const bool fields = out_pred || out_dir || out_cut;
  if ((rc = ensure_seeds(ctx, n)) != MNB_OK) return rc;
  // host-pointer staging, reserved before the workspace is sized; the single plan's outputs stay untouched for
  // mnb_cvp_backtrack / mnb_vector_map
  CallerArrays io(ctx);
  float* const o_matrix = mx ? io.out(mx->out, ctx->d_out_dist, (size_t)n * mx->m) : nullptr;
  float* const o_dist = io.out(out_dist, ctx->d_out_dist, rows);
  uint32_t* const o_pred = io.out(out_pred, ctx->d_batch_pred, rows);
  float* const o_dir = io.out(out_dir, ctx->d_batch_dir, rows);
  int32_t* const o_cut = io.out(out_cut, ctx->d_batch_cut, rows);
  CK(io.status());
  CvpMatrixArgs a{};
  auto prepare = [&](unsigned groups) -> int32_t {
    int32_t r;
    if ((r = ensure_workspace(ctx, groups)) != MNB_OK) return r;
    if (ctx->h_cancel) *ctx->h_cancel = 0;
    ctx->infl_labels_valid = false;            // the wavefront workspace is shared with the inflation wave
    CK(cudaMemcpyAsync(ctx->d_seed_faces, seed_faces, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_seed_pos, seed_pos, 3 * sizeof(float) * n, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(ctx->d_next_query, 0, sizeof(unsigned int), ctx->stream));
    CK(cudaMemsetAsync(ctx->ws.ctl, 0, sizeof(GroupCtl) * groups, ctx->stream));
    fill_cvp_args(ctx, a);
    a.n_queries = n; a.robot_face = -1; a.cost_limit = cost_limit; a.goal_dist_offset = 0.0;
    a.out_dist = o_dist; a.out_pred = o_pred; a.out_dir = o_dir; a.out_cut = o_cut;
    if (mx) {
      if ((r = upload_targets(ctx, *mx, a.tg)) != MNB_OK) return r;
      a.tg.out = o_matrix;
    }
    return MNB_OK;
  };
  const size_t per_group = ws_bytes_per_group(ctx->V);
  const CvpKernelArgs& b = a;
  unsigned groups = 1;
  rc = mx ? run_batch(ctx, [](auto c) { return k_cvp_batch<decltype(c)::value, false, CvpMatrixArgs>; }, a, n, per_group, ctx->ws_groups, "CVP", prepare, &groups)
     : fields ? run_batch(ctx, [](auto c) { return k_cvp_batch<decltype(c)::value, true>; }, b, n, per_group, ctx->ws_groups, "CVP", prepare, &groups)
              : run_batch(ctx, [](auto c) { return k_cvp_batch<decltype(c)::value, false>; }, b, n, per_group, ctx->ws_groups, "CVP", prepare, &groups);
  if (rc != MNB_OK) return rc;
  CK(io.copy_back());
  if ((rc = finish_stats(ctx, groups, 1)) != MNB_OK) return rc;
  if (ctx->h_cancel && *ctx->h_cancel) return MNB_CANCELED;
  return MNB_SUCCESS;
}

// mnb_cvp_batch_replan: mnb_cvp_batch_fields' rows for n goals, with the waves of the distinct goals resident in slots
// keyed by goal (DESIGN §4, "Batch replan").  Slots of goals absent from the call are released; a goal without one gets
// one while the cap and the device memory left after the workspace allow it.  A slot's wave resumes from its T0 when it
// holds the goal's wave of the same cost limit and cost generation (k_batch_replan_t0 decides the rest on the device).
static int32_t impl_cvp_batch_replan(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_faces, const float* seed_pos, double cost_limit,
                                     uint32_t n_changed, const uint32_t* changed, float* out_dist, uint32_t* out_pred, float* out_dir,
                                     int32_t* out_cut) {
  if (!ctx || !seed_faces || !seed_pos || (!out_dist && !out_pred && !out_dir && !out_cut) || !ctx->V || n == 0 || (n_changed && !changed))
    return MNB_E_ARG;
  const RepairRequest rq{n_changed, changed};
  int32_t rc;
  if ((rc = check_changed(ctx, &rq)) != MNB_OK) return rc;
  if (!ctx->costs_set) { ctx->err = "costs not set"; return MNB_E_STATE; }
  for (uint32_t i = 0; i < n; ++i) if (seed_faces[i] >= ctx->F) return MNB_INVALID_START;
  CK(cudaSetDevice(ctx->device));
  const uint32_t V = ctx->V, pool_cap = ws_pool_cap(V);
  const size_t slot_bytes = replan_slot_bytes(V, pool_cap);
  // the distinct goals in the order of their first row; key = seed face and the bits of the seed position
  using Key = std::array<uint32_t, 4>;
  std::map<Key, uint32_t> goal_index;
  std::vector<Key> keys; std::vector<uint32_t> goal_of(n), first;
  for (uint32_t i = 0; i < n; ++i) {
    Key k{seed_faces[i], 0, 0, 0};
    std::memcpy(&k[1], seed_pos + 3 * (size_t)i, 3 * sizeof(float));
    const auto it = goal_index.emplace(k, (uint32_t)keys.size());
    if (it.second) { keys.push_back(k); first.push_back(i); }
    goal_of[i] = it.first->second;
  }
  const uint32_t U = (uint32_t)keys.size();
  std::vector<uint32_t> u_faces(U); std::vector<float> u_pos(3 * (size_t)U);
  for (uint32_t u = 0; u < U; ++u) {
    u_faces[u] = seed_faces[first[u]];
    std::copy(seed_pos + 3 * (size_t)first[u], seed_pos + 3 * (size_t)first[u] + 3, &u_pos[3 * (size_t)u]);
  }
  uint64_t limit_bits;
  std::memcpy(&limit_bits, &cost_limit, sizeof(limit_bits));
  // release the slots of absent goals and those past the cap; other costs: the waves are stale
  std::vector<BatchReplanSlot>& slots = ctx->brs;
  const auto key_of = [](const BatchReplanSlot& s) { return Key{s.face, s.pos[0], s.pos[1], s.pos[2]}; };
  slots.erase(std::remove_if(slots.begin(), slots.end(), [&](const BatchReplanSlot& s) { return !goal_index.count(key_of(s)); }), slots.end());
  if (slots.size() > ctx->brs_max_slots) slots.resize(ctx->brs_max_slots);
  if (ctx->brs_cost_limit != limit_bits || ctx->brs_cost_gen != ctx->cost_gen)
    for (auto& sl : slots) sl.valid = false;
  std::vector<int64_t> slot_of(U, -1);
  for (size_t k = 0; k < slots.size(); ++k) slot_of[goal_index[key_of(slots[k])]] = (int64_t)k;
  if ((rc = ensure_seeds(ctx, U)) != MNB_OK) return rc;
  CallerArrays io(ctx);
  const size_t rows = (size_t)n * V;
  float* const o_dist = io.out(out_dist, ctx->d_out_dist, rows);
  uint32_t* const o_pred = io.out(out_pred, ctx->d_batch_pred, rows);
  float* const o_dir = io.out(out_dir, ctx->d_batch_dir, rows);
  int32_t* const o_cut = io.out(out_cut, ctx->d_batch_cut, rows);
  CK(io.status());
  CvpBatchReplanArgs a{};
  unsigned launches = 1;
  auto prepare = [&](unsigned groups) -> int32_t {
    int32_t r;
    if ((r = ensure_workspace(ctx, groups)) != MNB_OK) return r;
    // new slots: as many as the device memory left after the workspace allows, less the reserve batch_shape keeps
    size_t free_b = 0, total_b = 0;
    CK(device_memory(ctx->device, &free_b, &total_b));
    const size_t reserve = std::max<size_t>((size_t)512 << 20, total_b / 32);
    size_t room = free_b > reserve ? (free_b - reserve) / slot_bytes : 0;
    for (uint32_t u = 0; u < U && room > 0 && slots.size() < ctx->brs_max_slots; ++u) {
      if (slot_of[u] >= 0) continue;
      BatchReplanSlot sl;
      if (sl.mem.reserve(slot_bytes) != cudaSuccess) { (void)cudaGetLastError(); break; }
      sl.face = keys[u][0]; std::copy(&keys[u][1], &keys[u][1] + 3, sl.pos);
      slot_of[u] = (int64_t)slots.size();
      slots.push_back(std::move(sl));
      --room;
    }
    std::vector<BatchReplanGoal> table(U);
    bool any_resume = false;
    for (uint32_t u = 0; u < U; ++u) {
      BatchReplanGoal& t = table[u];
      t = BatchReplanGoal{};
      t.row = first[u];
      if (slot_of[u] >= 0) {
        const BatchReplanSlot& sl = slots[(size_t)slot_of[u]];
        t.slot = sl.mem.p;
        t.resume = sl.valid ? 1u : 0u;
        any_resume = any_resume || sl.valid;
      }
    }
    for (auto& sl : slots) sl.valid = false;     // until this call has succeeded
    CK(ctx->d_brs_goals.reserve(U));
    CK(cudaMemcpyAsync(ctx->d_brs_goals, table.data(), sizeof(BatchReplanGoal) * U, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_seed_faces, u_faces.data(), sizeof(uint32_t) * U, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_seed_pos, u_pos.data(), 3 * sizeof(float) * U, cudaMemcpyHostToDevice, ctx->stream));
    if (any_resume) {
      // T0 of the goals that may resume: chunks of the changed list per goal, about two blocks per SM in all
      const uint32_t chunks = std::max(1u, std::min((n_changed + 255u) / 256u, std::max(1u, 2u * (unsigned)ctx->sm_count / U)));
      CK(ctx->d_replan_chg.reserve(std::max(1u, n_changed))); CK(ctx->d_brs_minima.reserve(6 * (size_t)U * chunks));
      if (n_changed) CK(cudaMemcpyAsync(ctx->d_replan_chg, changed, sizeof(uint32_t) * n_changed, cudaMemcpyHostToDevice, ctx->stream));
      BatchReplanT0Args t{};
      t.V = V; t.pool_cap = pool_cap; t.faces = ctx->d_faces; t.cor_ptr = ctx->d_cor_ptr; t.cor_idx = ctx->d_cor_idx;
      t.goals = ctx->d_brs_goals; t.seed_faces = ctx->d_seed_faces; t.changed = ctx->d_replan_chg; t.n_changed = n_changed;
      t.chunks = chunks; t.minima = ctx->d_brs_minima;
      MNB_LAUNCH(k_batch_replan_t0, (size_t)U * chunks, 256, 0, ctx->stream, t);
      CK(cudaGetLastError());
      launches++;
    }
    if (ctx->h_cancel) *ctx->h_cancel = 0;
    ctx->infl_labels_valid = false;            // the wavefront workspace is shared with the inflation wave
    CK(cudaMemsetAsync(ctx->d_next_query, 0, sizeof(unsigned int), ctx->stream));
    CK(cudaMemsetAsync(ctx->ws.ctl, 0, sizeof(GroupCtl) * groups, ctx->stream));
    fill_cvp_args(ctx, a);
    a.n_queries = U; a.robot_face = -1; a.cost_limit = cost_limit; a.goal_dist_offset = 0.0;
    a.out_dist = o_dist; a.out_pred = o_pred; a.out_dir = o_dir; a.out_cut = o_cut;
    a.goals = ctx->d_brs_goals; a.pool_room = ctx->replan_pool_room;
    return MNB_OK;
  };
  unsigned groups = 1;
  rc = run_batch(ctx, [](auto c) { return k_cvp_batch_replan<decltype(c)::value>; }, a, U, ws_bytes_per_group(V), ctx->ws_groups, "CVP",
                 prepare, &groups);
  if (rc != MNB_OK) return rc;
  // duplicate goals: copies of their first row
  for (uint32_t i = 0; i < n; ++i) {
    const size_t src = (size_t)first[goal_of[i]] * V, dst = (size_t)i * V;
    if (src == dst) continue;
    if (o_dist) CK(cudaMemcpyAsync(o_dist + dst, o_dist + src, sizeof(float) * V, cudaMemcpyDeviceToDevice, ctx->stream));
    if (o_pred) CK(cudaMemcpyAsync(o_pred + dst, o_pred + src, sizeof(uint32_t) * V, cudaMemcpyDeviceToDevice, ctx->stream));
    if (o_dir) CK(cudaMemcpyAsync(o_dir + dst, o_dir + src, sizeof(float) * V, cudaMemcpyDeviceToDevice, ctx->stream));
    if (o_cut) CK(cudaMemcpyAsync(o_cut + dst, o_cut + src, sizeof(int32_t) * V, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  CK(io.copy_back());
  if ((rc = finish_stats(ctx, groups, launches)) != MNB_OK) return rc;
  if (ctx->h_cancel && *ctx->h_cancel) return MNB_CANCELED;
  for (auto& sl : slots) sl.valid = true;
  ctx->brs_cost_limit = limit_bits; ctx->brs_cost_gen = ctx->cost_gen;
  return MNB_SUCCESS;
}

static int32_t impl_dijkstra(mnb_ctx* ctx, uint32_t seed_vertex, int64_t robot_vertex, double cost_limit, double goal_dist_offset,
                     float* out_dist, uint32_t* out_pred) {
  if (!ctx || !ctx->V) return MNB_E_ARG;
  if (!ctx->costs_set) { ctx->err = "costs not set"; return MNB_E_STATE; }
  if (seed_vertex >= ctx->V) return MNB_INVALID_START;
  if (robot_vertex >= (int64_t)ctx->V) return MNB_INVALID_GOAL;
  CK(cudaSetDevice(ctx->device));
  int32_t rc;
  if ((rc = ensure_workspace(ctx, 1)) != MNB_OK) return rc;
  if ((rc = ensure_out(ctx, (size_t)ctx->V, true)) != MNB_OK) return rc;
  if (ctx->h_cancel) *ctx->h_cancel = 0;     // dijkstra:238
  ctx->infl_labels_valid = false;
  if ((rc = ensure_adj_tables(ctx)) != MNB_OK) return rc;
  CK(cudaMemsetAsync(ctx->ws.ctl, 0, sizeof(GroupCtl), ctx->stream));
  DijkstraKernelArgs a{};
  a.V = ctx->V; a.adj_ptr = ctx->d_adj_ptr; a.adj_nw = ctx->d_adj_nw; a.cost = ctx->d_cost;
  a.invalid = ctx->has_invalid ? ctx->d_invalid.p : nullptr; a.ws = wave_workspace(ctx); a.seed_vertex = seed_vertex;
  a.robot_vertex = robot_vertex; a.cost_limit = cost_limit; a.goal_dist_offset = goal_dist_offset; a.delta = ctx->delta;
  CallerArrays io(ctx);         // both rows are produced without the caller's arrays too: the outcome code reads them
  a.out_dist = io.needed(out_dist, ctx->d_out_dist.p, ctx->V);
  a.out_pred = io.needed(out_pred, ctx->d_out_pred.p, ctx->V);
  a.cancel_flag = ctx->d_cancel; a.max_rounds = watchdog_rounds(ctx->V);
  if (robot_vertex >= 0 && (uint32_t)robot_vertex == seed_vertex) {   // dijkstra:252-255: "start == goal" returns before the wave
    // the reference has cleared its maps by then (:241-249): distances +inf (seed 0), every vertex its own predecessor
    MNB_LAUNCH(k_dijkstra_trivial, (ctx->V + 255) / 256, 256, 0, ctx->stream, ctx->V, seed_vertex, a.out_dist, a.out_pred);
    CK(cudaGetLastError());
    CK(io.copy_back());
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->stats = mnb_stats{}; ctx->stats.kernel_launches = 1;
    return MNB_SUCCESS;
  }
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  cudaError_t e;
  const int cs = ctx->cluster;
  if (cs == -1) {   // single plan on the whole GPU (cooperative launch, one CTA per SM)
    a.delta = ctx->dijkstra_grid_delta; a.ell_adj = ctx->d_ell_adj; a.sweeps = ctx->sweeps; a.hop = ctx->w_mean > 0 ? 1.35f * ctx->w_mean : 0.16f;
    a.slots = ctx->grid_slots;
    size_t smem = 0;
    e = grid_kernel_smem(ctx, k_dijkstra_grid, 2, 512, smem);
    if (e == cudaSuccess) e = launch_cooperative(k_dijkstra_grid, a, (unsigned)ctx->sm_count, 512, ctx->stream, smem);
  } else {
    e = with_cluster_size<16>(cs, [&](auto c) {
      constexpr int CS = decltype(c)::value;
      return launch_cluster(k_dijkstra<CS>, a, CS, (unsigned)CS, ctx->threads, ctx->stream);
    });
  }
  if (e != cudaSuccess) { ctx->err = std::string("dijkstra launch: ") + cudaGetErrorString(e); return MNB_E_CUDA; }
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(io.copy_back());
  uint32_t rp = 0;
  if (robot_vertex >= 0) CK(cudaMemcpyAsync(&rp, a.out_pred + robot_vertex, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  if ((rc = finish_stats(ctx, 1, 1)) != MNB_OK) return rc;
  if (ctx->h_cancel && *ctx->h_cancel) return MNB_CANCELED;
  if (robot_vertex >= 0 && rp == (uint32_t)robot_vertex) return MNB_NO_PATH_FOUND;          // dijkstra:358-362
  return MNB_SUCCESS;
}

// n full-field Dijkstra waves in one launch (k_dijkstra_batch).  The waves run in a workspace of their own, so the
// results of the last mnb_cvp (predecessors, directions, cutting faces) and the labels of the last inflation stay valid.
// With mx (mnb_dijkstra_matrix; no row outputs) the waves run the matrix form k_dijkstra_batch<CS, true> into mx->out.
// With rq (mnb_dijkstra_batch_repair) out_dist / out_pred are the rows to repair (k_dijkstra_batch_repair<CS>), in place
// in device-pointer mode, through the device staging otherwise.
static int32_t impl_dijkstra_batch(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_vertices, double cost_limit, float* out_dist,
                                   uint32_t* out_pred, const MatrixRequest* mx = nullptr, const RepairRequest* rq = nullptr) {
  if (!ctx || !seed_vertices || (!out_dist && !out_pred && !mx) || !ctx->V || n == 0) return MNB_E_ARG;
  if (rq && (!out_dist || !out_pred || (rq->n && !rq->changed))) return MNB_E_ARG;
  int32_t rc;
  if ((rc = check_changed(ctx, rq)) != MNB_OK) return rc;
  if (!ctx->costs_set) { ctx->err = "costs not set"; return MNB_E_STATE; }
  for (uint32_t i = 0; i < n; ++i) if (seed_vertices[i] >= ctx->V) return MNB_INVALID_START;
  if ((rc = check_targets(ctx, mx)) != MNB_OK) return rc;
  if (rq && rq->n == 0) { ctx->stats = mnb_stats{}; return MNB_SUCCESS; }     // nothing changed: the rows are up to date
  CK(cudaSetDevice(ctx->device));
  const size_t V = ctx->V, rows = (size_t)n * V;
  if ((rc = ensure_seeds(ctx, n)) != MNB_OK) return rc;
  CallerArrays io(ctx);      // host-pointer staging, reserved before the workspace is sized
  float* const o_matrix = mx ? io.out(mx->out, ctx->d_out_dist, (size_t)n * mx->m) : nullptr;
  float* const o_dist = rq ? io.inout(out_dist, ctx->d_out_dist, rows) : io.out(out_dist, ctx->d_out_dist, rows);
  uint32_t* const o_pred = rq ? io.inout(out_pred, ctx->d_batch_pred, rows) : io.out(out_pred, ctx->d_batch_pred, rows);
  CK(io.status());
  DijkstraBatchArgs a{};
  DijkstraRepairArgs ra{};
  auto prepare = [&](unsigned groups) -> int32_t {
    int32_t r;
    if ((r = ensure_dijkstra_workspace(ctx, groups)) != MNB_OK) return r;
    if (ctx->h_cancel) *ctx->h_cancel = 0;     // dijkstra:238
    if ((r = ensure_adj_tables(ctx)) != MNB_OK) return r;
    CK(cudaMemcpyAsync(ctx->d_seed_faces, seed_vertices, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(ctx->d_next_query, 0, sizeof(unsigned int), ctx->stream));
    CK(cudaMemsetAsync(ctx->dws.ctl, 0, sizeof(GroupCtl) * groups, ctx->stream));
    a.V = ctx->V; a.adj_ptr = ctx->d_adj_ptr; a.adj_nw = ctx->d_adj_nw; a.cost = ctx->d_cost;
    a.invalid = ctx->has_invalid ? ctx->d_invalid.p : nullptr; a.ws = dijkstra_workspace(ctx);
    a.n_queries = n; a.seeds = ctx->d_seed_faces; a.cost_limit = cost_limit; a.delta = ctx->dijkstra_batch_delta;
    a.out_dist = o_dist; a.out_pred = o_pred;
    a.next_query = ctx->d_next_query; a.cancel_flag = ctx->d_cancel; a.max_rounds = watchdog_rounds(ctx->V);
    if (mx) {
      if ((r = upload_targets(ctx, *mx, a.tg)) != MNB_OK) return r;
      a.tg.out = o_matrix;
    }
    if (rq) {
      static_cast<DijkstraBatchArgs&>(ra) = a;
      if ((r = upload_changed(ctx, *rq, groups, ra.chg)) != MNB_OK) return r;
      // the repair resets the marks it sets; the batch kernel leaves its marks behind, a new workspace holds anything
      if (!ctx->dws_marks_clean) CK(cudaMemsetAsync(ctx->dws.mark, 0, sizeof(uint32_t) * (size_t)ctx->dws_groups * V, ctx->stream));
    }
    ctx->dws_marks_clean = false;
    return MNB_OK;
  };
  const size_t per_group = DIJKSTRA_BATCH_BYTES_PER_VERTEX * V + sizeof(GroupCtl);
  unsigned groups = 1;
  rc = rq ? run_batch(ctx, [](auto c) { return k_dijkstra_batch_repair<decltype(c)::value>; }, ra, n, per_group, ctx->dws_groups, "Dijkstra", prepare, &groups)
     : mx ? run_batch(ctx, [](auto c) { return k_dijkstra_batch<decltype(c)::value, true>; }, a, n, per_group, ctx->dws_groups, "Dijkstra", prepare, &groups)
          : run_batch(ctx, [](auto c) { return k_dijkstra_batch<decltype(c)::value>; }, a, n, per_group, ctx->dws_groups, "Dijkstra", prepare, &groups);
  if (rc != MNB_OK) return rc;
  CK(io.copy_back());
  if ((rc = finish_stats(ctx, groups, 1, ctx->dws.ctl)) != MNB_OK) return rc;
  ctx->dws_marks_clean = rq != nullptr;      // every wave of the repair has reset its marks (a canceled one too)
  if (ctx->h_cancel && *ctx->h_cancel) return MNB_CANCELED;
  return MNB_SUCCESS;
}

int32_t mnb_get_vertex_normals(mnb_ctx* ctx, float* out) {
  if (!ctx || !out || !ctx->V) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(CallerArrays(ctx).copy_out(out, ctx->d_vertex_normals.p, 3 * (size_t)ctx->V));
  CK(cudaStreamSynchronize(ctx->stream));
  return MNB_OK;
}

static int32_t impl_compute_layers(mnb_ctx* ctx, const mnb_layer_params* params, const float* clearance, float* out_costs,
                           float* out_combined, uint8_t* out_lethal_mask) {
  if (!ctx || !params || !ctx->V) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  const size_t V = ctx->V;
  CK(ctx->d_layer_costs.reserve(6 * V)); CK(ctx->d_layer_combined.reserve(V)); CK(ctx->d_layer_mask.reserve(V));
  CK(ctx->d_overflow.reserve(1));
  if (clearance) CK(ctx->d_clearance.reserve(V));
  CallerArrays io(ctx);
  const float* const d_clear = io.in(clearance, ctx->d_clearance.p, V);
  float* const o_costs = io.needed(out_costs, ctx->d_layer_costs.p, 6 * V);
  float* const o_combined = io.needed(out_combined, ctx->d_layer_combined.p, V);
  uint8_t* const o_mask = io.needed(out_lethal_mask, ctx->d_layer_mask.p, V);
  CK(io.status());
  CK(cudaMemsetAsync(ctx->d_overflow, 0, sizeof(unsigned int), ctx->stream));
  LayerKernelArgs a{};
  a.V = ctx->V; a.pos = ctx->d_pos; a.vn = ctx->d_vertex_normals; a.adj_ptr = ctx->d_adj_ptr; a.adj_nbr = ctx->d_adj_nbr;
  a.border = ctx->d_border; a.clearance = d_clear; a.P = *params;
  a.costs = o_costs; a.combined = o_combined; a.lethal_mask = o_mask;
  a.overflow = ctx->d_overflow;
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  if (ctx->layers_walk != LAYERS_WALK_LOCAL && !ctx->d_pos4) {
    CK(ctx->d_pos4.reserve(V)); CK(ctx->d_vn4.reserve(V)); CK(ctx->d_nbr8.reserve(8 * V));
    MNB_LAUNCH(k_pack_layers, (ctx->V + 255) / 256, 256, 0, ctx->stream, (const float*)ctx->d_pos, (const float*)ctx->d_vertex_normals,
               (const uint32_t*)ctx->d_adj_ptr, (const uint32_t*)ctx->d_adj_nbr, ctx->V, ctx->d_pos4, ctx->d_vn4, ctx->d_nbr8);
    CK(cudaGetLastError());
  }
  a.pos4 = ctx->d_pos4; a.vn4 = ctx->d_vn4; a.nbr8 = reinterpret_cast<const uint4*>(ctx->d_nbr8.p);
  const auto launch = [&](void (*kern)(const LayerKernelArgs), int threads, size_t smem) -> int32_t {
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MNB_LAUNCH(kern, (ctx->V + threads - 1) / threads, threads, smem, ctx->stream, a);
    return MNB_OK;
  };
  const int32_t rc = ctx->layers_walk == LAYERS_WALK_PF16 ? launch(k_layers<LAYERS_WALK_PF16>, PF_THREADS, PF_THREADS * SharedSeen<uint16_t>::BYTES)
                     : ctx->layers_walk == LAYERS_WALK_PF32 ? launch(k_layers<LAYERS_WALK_PF32>, PF_THREADS, PF_THREADS * SharedSeen<uint32_t>::BYTES)
                     : launch(k_layers<LAYERS_WALK_LOCAL>, LOCAL_THREADS, 0);
  if (rc != MNB_OK) return rc;
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(io.copy_back());
  unsigned int ovf = 0;
  CK(cudaMemcpyAsync(&ovf, ctx->d_overflow, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  simple_stats(ctx, 1, ctx->V);
  if (ovf) { ctx->err = "layer neighbourhood exceeds the per-vertex scratch (radius too large for the mesh resolution)"; return MNB_E_NOMEM; }
  return MNB_OK;
}

static int32_t impl_vector_map(mnb_ctx* ctx, const uint32_t* pred, const float* direction, const int32_t* cutting_face, float* out_vec) {
  if (!ctx || !ctx->V || !out_vec) return MNB_E_ARG;
  if (!pred && !ctx->last_valid) { ctx->err = "mnb_vector_map(pred = NULL) needs a successful mnb_cvp on this context first"; return MNB_E_STATE; }
  CK(cudaSetDevice(ctx->device));
  const size_t V = ctx->V;
  CallerArrays io(ctx);
  DeviceBuffer<float> tmp_out, tmp_dir; DeviceBuffer<uint32_t> tmp_pred; DeviceBuffer<int32_t> tmp_cut;
  float* const d_out = io.out(out_vec, tmp_out, 3 * V);
  // pred NULL: the device-resident result of the last CVP plan (nothing is uploaded)
  const uint32_t* const d_pred = pred ? io.in(pred, tmp_pred, V) : ctx->last_pred;
  const float* const d_dir = pred ? io.in(direction, tmp_dir, V) : ctx->last_dir;
  const int32_t* const d_cut = pred ? io.in(cutting_face, tmp_cut, V) : ctx->last_cut;
  CK(io.status());
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  MNB_LAUNCH(k_vector_map, (ctx->V + 255) / 256, 256, 0, ctx->stream, ctx->d_pos, ctx->d_vertex_normals, d_pred, d_dir, d_cut, ctx->V, d_out);
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(io.copy_back());
  CK(cudaStreamSynchronize(ctx->stream));
  simple_stats(ctx, 1, ctx->V);
  return MNB_OK;
}

static int32_t impl_cvp_backtrack(mnb_ctx* ctx, const float robot_pos[3], uint32_t robot_face, double step_width, uint32_t max_points,
                          float* path_pos, uint32_t* path_face, uint32_t* n_points) {
  if (!ctx || !ctx->V || !robot_pos || !path_pos || !n_points || max_points < 2) return MNB_E_ARG;
  if (!ctx->last_valid) { ctx->err = "mnb_cvp_backtrack needs a preceding successful mnb_cvp on this context"; return MNB_E_STATE; }
  if (robot_face >= ctx->F) return MNB_INVALID_GOAL;
  CK(cudaSetDevice(ctx->device));
  CK(ctx->d_path_pos.reserve(3 * (size_t)max_points)); CK(ctx->d_path_face.reserve(max_points));
  CK(ctx->d_bt_result.reserve(2));
  uint32_t n = 0;           // points written: read back after the launch
  CallerArrays io(ctx);
  BacktrackArgs a{};
  a.pos = ctx->d_pos; a.vn = ctx->d_vertex_normals; a.faces = ctx->d_faces; a.cor_ptr = ctx->d_cor_ptr; a.cor_idx = ctx->d_cor_idx;
  a.pred = ctx->last_pred; a.direction = ctx->last_dir; a.cut = ctx->last_cut;
  for (int k = 0; k < 3; ++k) { a.start[k] = ctx->last_seed_pos[k]; a.goal[k] = robot_pos[k]; }
  a.start_face = ctx->last_seed_face; a.goal_face = robot_face; a.step_width = step_width; a.max_points = max_points;
  a.path_pos = io.out(path_pos, ctx->d_path_pos.p, 3, &n); a.path_face = io.needed(path_face, ctx->d_path_face.p, 1, &n); a.result = ctx->d_bt_result; a.cancel_flag = ctx->d_cancel;
  a.layer = RepulsiveField{};
  if (ctx->repulsive_on && ctx->infl_field_valid) a.layer = repulsive_field_of(ctx);
  CK(cudaFuncSetAttribute(k_backtrack, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BtShared)));
  int32_t res[2] = {0, 0};
  for (;;) {
    a.spill_list = ctx->d_bt_spill_list; a.spill_key = ctx->d_bt_spill_key;
    CK(cudaEventRecord(ctx->ev0, ctx->stream));
    MNB_LAUNCH(k_backtrack, 1, 32, sizeof(BtShared), ctx->stream, a);
    CK(cudaGetLastError());
    CK(cudaEventRecord(ctx->ev1, ctx->stream));
    CK(cudaMemcpyAsync(res, ctx->d_bt_result, sizeof(res), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (res[0] != BT_NEEDS_SPILL) break;
    // a face search outgrew shared memory: reserve the unbounded one (keys all zero) and walk again -- the walk is
    // deterministic, so the second one returns what one walk with the workspace would
    CK(ctx->d_bt_spill_list.reserve(ctx->F)); CK(ctx->d_bt_spill_key.reserve(ctx->F));
    CK(cudaMemsetAsync(ctx->d_bt_spill_key, 0, sizeof(uint32_t) * (size_t)ctx->F, ctx->stream));
  }
  n = (uint32_t)res[1] < max_points ? (uint32_t)res[1] : max_points;
  *n_points = n;
  CK(io.copy_back());
  CK(cudaStreamSynchronize(ctx->stream));
  simple_stats(ctx, 1, n);
  if (res[0] == MNB_E_STATE) { ctx->err = "back-tracking exceeded max_points (cyclic vector field?)"; return MNB_E_STATE; }
  return res[0];
}

static int32_t impl_locate(mnb_ctx* ctx, uint32_t n, const float* points, uint32_t* out_vertex, int32_t* out_face, float* out_bary) {
  if (!ctx || !ctx->V || !points || n == 0) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  DeviceBuffer<float> d_pts, d_b; DeviceBuffer<unsigned long long> d_keys; DeviceBuffer<uint32_t> d_v; DeviceBuffer<int32_t> d_f;
  CK(d_keys.reserve((size_t)n));
  CK(cudaMemsetAsync(d_keys, 0xff, sizeof(unsigned long long) * (size_t)n, ctx->stream));
  CallerArrays io(ctx);
  const float* const pts = io.in(points, d_pts, 3 * (size_t)n);
  uint32_t* const o_vertex = io.out(out_vertex, d_v, n);
  int32_t* const o_face = io.out(out_face, d_f, n);
  float* const o_bary = io.out(out_bary, d_b, 3 * (size_t)n);
  CK(io.status());
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  const uint32_t want = (ctx->V + 255) / 256, cap = (uint32_t)ctx->sm_count * 8;
  const uint32_t blocks = want < cap ? want : cap;
  uint32_t launches = 0;
  for (uint32_t q0 = 0; q0 < n; q0 += LOC_Q, ++launches)
    MNB_LAUNCH(k_nearest_vertex, blocks, 256, 0, ctx->stream, ctx->d_pos, ctx->V, pts, q0, n - q0 < (uint32_t)LOC_Q ? n - q0 : (uint32_t)LOC_Q, d_keys);
  MNB_LAUNCH(k_containing_face, (n + 127) / 128, 128, 0, ctx->stream, ctx->d_pos, ctx->d_faces, ctx->d_cor_ptr, ctx->d_cor_idx, pts, n, d_keys,
             o_vertex, o_face, o_bary);
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(io.copy_back());
  CK(cudaStreamSynchronize(ctx->stream));
  simple_stats(ctx, launches + 1, n);
  return MNB_OK;
}

// experiment knob (not part of the public header): in-round sweeps of the whole-grid single-plan kernel
int32_t mnb_debug_set_sweeps(mnb_ctx* ctx, int32_t k) { if (!ctx || k < -1 || k > 64) return MNB_E_ARG; ctx->sweeps = k; return MNB_OK; }

// test hook (not part of the public header): GridStage slots per CTA of the whole-grid single-plan kernels, 1 up to what the
// device's shared memory holds (0 = the default).  The band widths derived from the slots follow at the next mnb_set_costs.
int32_t mnb_debug_set_sweep_slots(mnb_ctx* ctx, int32_t n) {
  if (!ctx || n < 0 || (uint32_t)n > ctx->grid_slots_max) return MNB_E_ARG;
  ctx->grid_slots = n ? (uint32_t)n : std::min(GRID_SLOTS_DEFAULT, ctx->grid_slots_max);
  ctx->grid_blocks_per_sm = 0;
  return MNB_OK;
}

// test hook (not part of the public header): a resumed replan wave may add at most `words` level-pool words (0 = no limit
// but the pool's), so that tests reach the whole-wave retry after a resumed wave ran out of pool
int32_t mnb_debug_set_replan_pool_room(mnb_ctx* ctx, uint32_t words) { if (!ctx) return MNB_E_ARG; ctx->replan_pool_room = words; return MNB_OK; }
// the most resident slots mnb_cvp_batch_replan keeps (n < 0: no cap but the device memory); slots past it are released by
// the next call
int32_t mnb_debug_set_batch_replan_slots(mnb_ctx* ctx, int32_t n) {
  if (!ctx) return MNB_E_ARG;
  ctx->brs_max_slots = n < 0 ? 0xffffffffu : (uint32_t)n;
  return MNB_OK;
}
// the resident slots of mnb_cvp_batch_replan and how many of them hold a wave the next call may resume
int32_t mnb_debug_get_batch_replan_slots(mnb_ctx* ctx, uint32_t* n_slots, uint32_t* n_valid) {
  if (!ctx || !n_slots || !n_valid) return MNB_E_ARG;
  *n_slots = (uint32_t)ctx->brs.size();
  *n_valid = (uint32_t)std::count_if(ctx->brs.begin(), ctx->brs.end(), [](const BatchReplanSlot& s) { return s.valid; });
  return MNB_OK;
}

int32_t mnb_debug_set_infl_skip(mnb_ctx* ctx, int32_t on) { if (!ctx) return MNB_E_ARG; ctx->infl_skip_clean = on != 0; return MNB_OK; }
int32_t mnb_debug_set_layers_smem(mnb_ctx* ctx, int32_t mode) {
  if (!ctx || (mode != LAYERS_WALK_LOCAL && mode != LAYERS_WALK_PF32 && mode != LAYERS_WALK_PF16)) return MNB_E_ARG;
  ctx->layers_walk = mode; ctx->layers_explicit = true; return MNB_OK;
}

// test hooks (not part of the public header) of the single-plan CVP epilogue.  set: 0 (default) replays a vertex on its
// ELL row where that covers it and hands the others to the CSR replay; 1 hands every vertex that is replayed at all (reached,
// eligible, not a seed) to the CSR replay, so that tests can compare the two on the same labels.  get: the number of
// vertices the last single plan's epilogue handed to the CSR replay (ctl->epi_csr of the workspace it ran on: the
// resident one for mnb_cvp_replan)
int32_t mnb_debug_set_cvp_epilogue(mnb_ctx* ctx, int32_t mode) { if (!ctx || mode < 0 || mode > 1) return MNB_E_ARG; ctx->cvp_epilogue = mode; return MNB_OK; }
int32_t mnb_debug_get_epilogue_csr(mnb_ctx* ctx, uint32_t* n) {
  if (!ctx || !n) return MNB_E_ARG;
  const GroupCtl* ctl = ctx->epi_in_rw ? ctx->rw.ctl.p : ctx->ws.ctl.p;
  if (!ctl) return MNB_E_STATE;
  CK(cudaMemcpy(n, &ctl->epi_csr, sizeof(uint32_t), cudaMemcpyDeviceToHost));
  return MNB_OK;
}

// debugging aid (not part of the public header): raw labels {d, a1, a2, a3|flag} of wavefront group 0
int32_t mnb_debug_get_labels(mnb_ctx* ctx, uint32_t* out4v) {
  if (!ctx || !ctx->ws.state) return MNB_E_ARG;
  CK(cudaMemcpy(out4v, ctx->ws.state, sizeof(uint4) * (size_t)ctx->V, cudaMemcpyDeviceToHost));
  return MNB_OK;
}

// debugging aid (not part of the public header): side arrays of the labels of wavefront group 0 (level-1 ids, ext words,
// the first n_pool words of the level pool) -- tools/emu_pop_order.py rebuilds every vertex' level stack from them
int32_t mnb_debug_get_label_sides(mnb_ctx* ctx, uint32_t* root, uint32_t* ext, uint32_t* pool, uint32_t n_pool) {
  if (!ctx || !ctx->ws.state) return MNB_E_ARG;
  CK(cudaMemcpy(root, ctx->ws.root, sizeof(uint32_t) * (size_t)ctx->V, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(ext, ctx->ws.ext, sizeof(uint32_t) * (size_t)ctx->V, cudaMemcpyDeviceToHost));
  if (n_pool) CK(cudaMemcpy(pool, ctx->ws.pool, sizeof(uint32_t) * (size_t)std::min<uint32_t>(n_pool, ws_pool_cap(ctx->V)), cudaMemcpyDeviceToHost));
  return MNB_OK;
}

}  // extern "C"

// The inputs of an inflation wave: the workspace, the scratch outputs, the lethal list and the invalid mask staged into
// d_lethals / d_invalid (device copies of the caller's arrays in either pointer mode).
static int32_t stage_inflation(mnb_ctx* ctx, const uint32_t* lethals, uint32_t n, const uint8_t* invalid,
                               DeviceBuffer<uint32_t>& d_lethals, DeviceBuffer<uint8_t>& d_invalid) {
  int32_t rc;
  if ((rc = ensure_workspace(ctx, 1)) != MNB_OK) return rc;
  if ((rc = ensure_out(ctx, (size_t)ctx->V, false)) != MNB_OK) return rc;
  CK(ctx->d_out_cost.reserve(ctx->V));
  CallerArrays io(ctx);
  CK(d_lethals.reserve(n));
  if (n) CK(io.copy_in(d_lethals.p, lethals, n));
  if (invalid) {
    CK(d_invalid.reserve(ctx->V));
    CK(io.copy_in(d_invalid.p, invalid, ctx->V));
  }
  return MNB_OK;
}

// one k_inflate launch from a device lethal list (ev0 is recorded just before it when record_start is set)
static int32_t launch_inflate(mnb_ctx* ctx, const uint32_t* d_lethals, uint32_t n, const uint8_t* d_invalid,
                              const mnb_inflation_params* params, float* out_dist, float* out_cost, bool record_start) {
  CK(cudaMemsetAsync(ctx->ws.ctl, 0, sizeof(GroupCtl), ctx->stream));
  InflateKernelArgs a{};
  a.V = ctx->V; a.cor_ptr = ctx->d_cor_ptr; a.cor_idx = ctx->d_cor_idx; a.cor_wd = ctx->d_cor_wd; a.cor_eid = ctx->d_cor_eid;
  a.invalid = d_invalid; a.ws = wave_workspace(ctx); a.lethals = d_lethals; a.n_lethals = n;
  a.max_distance = (float)params->inflation_radius;      // double -> `const float&` parameter (inflation_layer.cpp:240,450)
  a.params.inscribed_radius = params->inscribed_radius; a.params.inflation_radius = params->inflation_radius;
  a.params.lethal_value = params->lethal_value; a.params.inscribed_value = params->inscribed_value;
  a.params.cost_scaling_factor = params->cost_scaling_factor;
  a.out_dist = out_dist; a.out_cost = out_cost;
  a.max_rounds = watchdog_rounds(ctx->V); a.skip_clean = ctx->infl_skip_clean;
  if (record_start) CK(cudaEventRecord(ctx->ev0, ctx->stream));
  int infl_per_sm = 1;
  if (MNB_INFL_MINBLOCKS > 1) {
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&infl_per_sm, k_inflate, ctx->threads, 0));
    infl_per_sm = std::max(1, std::min(infl_per_sm, (int)MNB_INFL_MINBLOCKS));
  }
  CK(launch_cooperative(k_inflate, a, (unsigned)(ctx->sm_count * infl_per_sm), ctx->threads, ctx->stream));
  return MNB_OK;
}

// InflationLayer::waveCostInflation; with want_update additionally the update set of InflationLayer::onInputChanged
static int32_t inflate_impl(mnb_ctx* ctx, const uint32_t* lethals, uint32_t n, const uint8_t* invalid,
                            const mnb_inflation_params* params, float* out_dist, float* out_cost, bool want_update,
                            uint32_t* out_changed, uint32_t* n_changed) {
  if (!ctx || !ctx->V || !params || (n && !lethals)) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  ctx->infl_labels_valid = false;
  ctx->infl_resident = false; ctx->infl_cid_valid = false; ctx->infl_field_resident = false;
  int32_t rc;
  if ((rc = stage_inflation(ctx, lethals, n, invalid, ctx->d_lethals, ctx->d_infl_invalid)) != MNB_OK) return rc;
  // both outputs are produced without the caller's arrays too: they become the resident distances and riskiness
  CallerArrays io(ctx);
  float* const o_dist = io.needed(out_dist, ctx->d_out_dist.p, ctx->V);
  float* const o_cost = io.needed(out_cost, ctx->d_out_cost.p, ctx->V);
  if ((rc = launch_inflate(ctx, ctx->d_lethals, n, invalid ? ctx->d_infl_invalid.p : nullptr, params, o_dist, o_cost, true)) != MNB_OK) return rc;
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(io.copy_back());
  int32_t rc2 = finish_stats(ctx, 1, 1);
  if (rc2 != MNB_OK) return rc2;
  // the riskiness map of this run is the "previous" one of the next mnb_inflation_update (riskiness_ = std::move(new_costs))
  const size_t V = ctx->V;
  if (want_update) {
    const uint32_t n_tiles = (uint32_t)((V + US_TILE - 1) / US_TILE);
    CK(ctx->d_changed.reserve(V)); CK(ctx->d_tile_count.reserve(n_tiles)); CK(ctx->d_total.reserve(1));
    const float* old = ctx->prev_risk_valid ? ctx->d_prev_risk.p : nullptr;
    unsigned int total = 0;
    uint32_t* const d_out = io.needed(out_changed, ctx->d_changed.p, 1, &total);
    MNB_LAUNCH(k_update_set_count, n_tiles, 256, 0, ctx->stream, (const float*)o_cost, old, ctx->V, ctx->d_tile_count);
    MNB_LAUNCH(k_update_set_scan, 1, 1024, 0, ctx->stream, ctx->d_tile_count, n_tiles, ctx->d_total);
    MNB_LAUNCH(k_update_set_write, n_tiles, 256, 0, ctx->stream, (const float*)o_cost, old, ctx->V, (const unsigned int*)ctx->d_tile_count, d_out);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(&total, ctx->d_total, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (n_changed) *n_changed = total;
    CK(io.copy_back());
    ctx->stats.kernel_launches += 3;
  }
  CK(ctx->d_prev_risk.reserve(V));
  CK(cudaMemcpyAsync(ctx->d_prev_risk, o_cost, sizeof(float) * V, cudaMemcpyDeviceToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->prev_risk_valid = true;
  ctx->infl_labels_valid = true; ctx->infl_had_invalid = invalid != nullptr; ctx->infl_params = *params; ctx->infl_field_valid = false; ctx->infl_rounds = ctx->stats.rounds;
  CK(ctx->d_infl_dist.reserve(V));
  CK(cudaMemcpyAsync(ctx->d_infl_dist, o_dist, sizeof(float) * V, cudaMemcpyDeviceToDevice, ctx->stream));   // distances_
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->infl_resident = true; ctx->infl_n_lethals = n;
  return MNB_OK;
}

// mnb_inflation_repair (DESIGN §4): a fresh inflation wave from the lethals of the clusters of the resident result that
// the change can reach, patched into the resident result; everything outside those clusters and the new footprint keeps
// its bits.  Without a resident result, or with other parameters than it was computed with: one whole-map wave.
static int32_t impl_inflation_repair(mnb_ctx* ctx, const uint32_t* lethals, uint32_t n, const uint8_t* invalid,
                                     const mnb_inflation_params* params, float* out_dist, float* out_cost,
                                     uint32_t* out_changed, uint32_t* n_changed) {
  if (!ctx || !ctx->V || !params || (n && !lethals) || !n_changed) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  const uint32_t V = ctx->V, W = V / 32 + 1;
  const bool local = ctx->infl_resident && std::memcmp(params, &ctx->infl_params, sizeof(mnb_inflation_params)) == 0;
  const bool field = ctx->infl_field_valid, has_risk = ctx->prev_risk_valid, labels = ctx->infl_labels_valid;
  ctx->infl_labels_valid = false;
  int32_t rc;
  if ((rc = stage_inflation(ctx, lethals, n, invalid, ctx->d_infl_lethals_next, ctx->d_infl_invalid_next)) != MNB_OK) return rc;
  CK(ctx->d_infl_bits.reserve(4 * (size_t)W)); CK(ctx->d_infl_cnt.reserve(6));
  CK(ctx->d_infl_seeds.reserve(std::max(n, 1u))); CK(ctx->d_infl_region.reserve(V));
  CK(ctx->d_infl_dist.reserve(V)); CK(ctx->d_prev_risk.reserve(V)); CK(ctx->d_infl_cid.reserve(V));
  const uint32_t n_tiles = (W + BITS_TILE_WORDS - 1) / BITS_TILE_WORDS;
  CK(ctx->d_changed.reserve(V)); CK(ctx->d_tile_count.reserve(n_tiles)); CK(ctx->d_total.reserve(1));
  // from here on the resident result is being rewritten: a failure leaves none
  ctx->infl_resident = false; ctx->prev_risk_valid = false; ctx->infl_field_valid = false; ctx->infl_field_resident = false;
  uint32_t* const old_bits = ctx->d_infl_bits; uint32_t* const new_bits = old_bits + W;
  uint32_t* const aff = old_bits + 2 * (size_t)W; uint32_t* const chg = old_bits + 3 * (size_t)W;
  unsigned int* const d_cnt = ctx->d_infl_cnt;
  const uint8_t* const new_inv = invalid ? ctx->d_infl_invalid_next.p : nullptr;
  // the changed list, then the dense outputs of a wave: without a wave the outputs are copies of the resident arrays
  unsigned int total = 0;
  CallerArrays list(ctx), rows(ctx);
  uint32_t* const d_out = list.needed(out_changed, ctx->d_changed.p, 1, &total);
  float* const o_dist = rows.needed(out_dist, ctx->d_out_dist.p, V);
  float* const o_cost = rows.needed(out_cost, ctx->d_out_cost.p, V);
  CK(cudaMemsetAsync(old_bits, 0, sizeof(uint32_t) * 4 * (size_t)W, ctx->stream));
  CK(cudaMemsetAsync(d_cnt, 0, 6 * sizeof(unsigned int), ctx->stream));
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  uint64_t launches = 0, rounds = 0, recomputes = 0, settled = 0, skipped = 0, last_rounds = 0;
  unsigned int cnt[6] = {0u, 0u, 0u, 0u, 0u, 0u};
  auto read_cnt = [&]() -> int32_t {
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(cnt, d_cnt, sizeof(cnt), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return MNB_OK;
  };
  auto wave = [&](const uint32_t* seeds, uint32_t ns) -> int32_t {   // one pass: k_inflate from `seeds`
    int32_t r = launch_inflate(ctx, seeds, ns, new_inv, params, o_dist, o_cost, false);
    if (r != MNB_OK) return r;
    CK(cudaEventRecord(ctx->ev1, ctx->stream));
    if ((r = finish_stats(ctx, 1, 1)) != MNB_OK) return r;
    rounds += ctx->stats.rounds; recomputes += ctx->stats.recomputes; settled += ctx->stats.settled; skipped += ctx->stats.skipped;
    last_rounds = ctx->stats.rounds; ++launches;
    return MNB_OK;
  };
  bool ran = true;                           // a wave ran: o_dist / o_cost hold its dense output
  bool whole = !local;                       // the wave is the whole-map one
  uint32_t n_region = 0;
  ClusterArgs ca{};
  ca.V = V; ca.cor_ptr = ctx->d_cor_ptr; ca.cor_idx = ctx->d_cor_idx; ca.dist = ctx->d_infl_dist; ca.cid = ctx->d_infl_cid;
  if (local) {
    if (!ctx->infl_cid_valid) {              // the first repair after a whole-map wave: cluster ids of its footprint
      MNB_LAUNCH(k_cluster_init, (V + 255) / 256, 256, 0, ctx->stream, ca);
      MNB_LAUNCH(k_cluster_unite, (V + 255) / 256, 256, 0, ctx->stream, ca);
      MNB_LAUNCH(k_cluster_flatten, (V + 255) / 256, 256, 0, ctx->stream, ca);
      launches += 3;
    }
    ctx->infl_cid_valid = false;
    InflRepairArgs ra{};
    ra.V = V; ra.cor_ptr = ctx->d_cor_ptr; ra.cor_idx = ctx->d_cor_idx; ra.cid = ctx->d_infl_cid;
    ra.old_bits = old_bits; ra.new_bits = new_bits; ra.old_inv = ctx->infl_had_invalid ? ctx->d_infl_invalid.p : nullptr; ra.new_inv = new_inv;
    ra.aff = aff; ra.lethals = ctx->d_infl_lethals_next; ra.n_lethals = n; ra.seeds = ctx->d_infl_seeds; ra.cnt = d_cnt;
    if (ctx->infl_n_lethals) { MNB_LAUNCH(k_lethal_bits, (ctx->infl_n_lethals + 255) / 256, 256, 0, ctx->stream, (const uint32_t*)ctx->d_lethals, ctx->infl_n_lethals, V, old_bits); ++launches; }
    if (n) { MNB_LAUNCH(k_lethal_bits, (n + 255) / 256, 256, 0, ctx->stream, (const uint32_t*)ctx->d_infl_lethals_next, n, V, new_bits); ++launches; }
    MNB_LAUNCH(k_infl_delta, (V + 255) / 256, 256, 0, ctx->stream, ra);
    MNB_LAUNCH(k_infl_affected_count, (V + 255) / 256, 256, 0, ctx->stream, ra);
    launches += 2;
    if ((rc = read_cnt()) != MNB_OK) return rc;
    ran = cnt[0] != 0;                       // nothing changed: no wave
    whole = ran && (double)cnt[5] > INFL_REPAIR_MAX_SHARE * (double)cnt[4];
    // passes: the seeds of the affected clusters, their wave, the merge check; a new footprint that touches an unaffected
    // cluster makes it affected, so the set of affected clusters only grows and the loop ends
    for (bool again = ran && !whole; again;) {
      CK(cudaMemsetAsync(d_cnt + 1, 0, 2 * sizeof(unsigned int), ctx->stream));
      if (n) { MNB_LAUNCH(k_infl_seeds, (n + 255) / 256, 256, 0, ctx->stream, ra); ++launches; }
      if ((rc = read_cnt()) != MNB_OK) return rc;
      if ((rc = wave(ctx->d_infl_seeds, cnt[1])) != MNB_OK) return rc;
      MNB_LAUNCH(k_infl_merge_check, (V + 255) / 256, 256, 0, ctx->stream, ra, (const float*)o_dist);
      ++launches;
      if ((rc = read_cnt()) != MNB_OK) return rc;
      again = cnt[2] != 0;
    }
  }
  if (whole && (rc = wave(ctx->d_infl_lethals_next, n)) != MNB_OK) return rc;
  if (ran) {
    InflPatchArgs pa{};
    pa.V = V; pa.all = whole ? 1 : 0; pa.aff = aff; pa.cid = whole ? nullptr : ctx->d_infl_cid.p;
    pa.out_dist = o_dist; pa.out_cost = o_cost; pa.res_dist = ctx->d_infl_dist; pa.res_risk = ctx->d_prev_risk;
    pa.has_risk = local || has_risk; pa.chg_bits = chg; pa.region = ctx->d_infl_region; pa.n_region = d_cnt + 3;
    MNB_LAUNCH(k_infl_patch, (V + 255) / 256, 256, 0, ctx->stream, pa);
    ++launches;
    if ((rc = read_cnt()) != MNB_OK) return rc;
    n_region = cnt[3];
    if (!whole && n_region) {                // cluster ids of the region: the components of the new footprint
      ca.list = ctx->d_infl_region; ca.n = n_region;
      MNB_LAUNCH(k_cluster_unite, (n_region + 255) / 256, 256, 0, ctx->stream, ca);
      MNB_LAUNCH(k_cluster_flatten, (n_region + 255) / 256, 256, 0, ctx->stream, ca);
      launches += 2;
    }
    ctx->infl_cid_valid = !whole;
  } else {
    ctx->infl_cid_valid = true;
  }
  // the changed set: ordered compaction of the bits the patch set
  MNB_LAUNCH(k_bits_count, n_tiles, 256, 0, ctx->stream, (const uint32_t*)chg, W, ctx->d_tile_count);
  MNB_LAUNCH(k_update_set_scan, 1, 1024, 0, ctx->stream, ctx->d_tile_count, n_tiles, ctx->d_total);
  MNB_LAUNCH(k_bits_write, n_tiles, 256, 0, ctx->stream, (const uint32_t*)chg, W, (const unsigned int*)ctx->d_tile_count, d_out);
  launches += 3;
  CK(cudaGetLastError());
  // the new set and mask are the resident ones from here on
  std::swap(ctx->d_lethals, ctx->d_infl_lethals_next);
  if (invalid) std::swap(ctx->d_infl_invalid, ctx->d_infl_invalid_next);
  ctx->infl_n_lethals = n; ctx->infl_had_invalid = invalid != nullptr; ctx->infl_params = *params;
  if (ran) ctx->infl_rounds = last_rounds;
  // a whole-map wave leaves whole-map labels in the workspace; without a wave the labels there are still current
  ctx->infl_labels_valid = whole || (!ran && labels);
  if (field && ran && (whole || n_region)) {   // the repulsive field of the region (of every vertex after a whole-map wave)
    unsigned fl = 0;
    if ((rc = infl_vector_field(ctx, whole ? nullptr : ctx->d_infl_region.p, n_region, fl)) != MNB_OK) return rc;
    launches += fl;
  }
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(cudaMemcpyAsync(&total, ctx->d_total, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  *n_changed = total;
  CK(list.copy_back());
  if (ran) {
    CK(rows.copy_back());
  } else {
    if (out_dist) CK(rows.copy_out(out_dist, ctx->d_infl_dist.p, V));
    if (out_cost) CK(rows.copy_out(out_cost, ctx->d_prev_risk.p, V));
  }
  CK(cudaStreamSynchronize(ctx->stream));
  float ms = 0; cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
  ctx->stats = mnb_stats{};
  ctx->stats.rounds = rounds; ctx->stats.recomputes = recomputes; ctx->stats.settled = settled; ctx->stats.skipped = skipped;
  ctx->stats.kernel_launches = launches; ctx->stats.kernel_ms = ms;
  ctx->infl_resident = true; ctx->prev_risk_valid = true;
  ctx->infl_field_valid = field; ctx->infl_field_resident = field;
  return MNB_OK;
}

extern "C" {

static int32_t impl_inflate(mnb_ctx* ctx, const uint32_t* lethals, uint32_t n, const uint8_t* invalid,
                    const mnb_inflation_params* params, float* out_dist, float* out_cost) {
  return inflate_impl(ctx, lethals, n, invalid, params, out_dist, out_cost, false, nullptr, nullptr);
}

static int32_t impl_inflation_update(mnb_ctx* ctx, const uint32_t* lethals, uint32_t n, const uint8_t* invalid,
                             const mnb_inflation_params* params, float* out_dist, float* out_cost, uint32_t* out_changed,
                             uint32_t* n_changed) {
  if (!n_changed) return MNB_E_ARG;
  return inflate_impl(ctx, lethals, n, invalid, params, out_dist, out_cost, true, out_changed, n_changed);
}

int32_t mnb_get_costs(mnb_ctx* ctx, float* out_vertex_costs, float* out_edge_weights) {
  if (!ctx || !ctx->V) return MNB_E_ARG;
  if (!ctx->costs_set) { ctx->err = "costs not set"; return MNB_E_STATE; }
  CK(cudaSetDevice(ctx->device));
  CallerArrays io(ctx);
  if (out_vertex_costs) CK(io.copy_out(out_vertex_costs, ctx->d_cost.p, ctx->V));
  if (out_edge_weights) CK(io.copy_out(out_edge_weights, ctx->d_edge_w.p, ctx->E));
  CK(cudaStreamSynchronize(ctx->stream));
  return MNB_OK;
}

static int32_t impl_update_vertex_costs(mnb_ctx* ctx, uint32_t n_changed, const uint32_t* changed, const float* costs,
                                int32_t costs_indexed_by_vertex, float default_value, double edge_cost_factor) {
  if (!ctx || !ctx->V || (n_changed && (!changed || !costs))) return MNB_E_ARG;
  if (!ctx->costs_set) { ctx->err = "mnb_update_vertex_costs needs mnb_set_costs / mnb_compute_edge_weights first"; return MNB_E_STATE; }
  if (n_changed == 0) return MNB_OK;
  CK(cudaSetDevice(ctx->device));
  CallerArrays io(ctx);
  const uint32_t* const d_ids = io.in(changed, ctx->d_upd_ids, n_changed);
  const float* const d_costs = io.in(costs, ctx->d_upd_costs, costs_indexed_by_vertex ? (size_t)ctx->V : (size_t)n_changed);
  CK(io.status());
  if (!ctx->d_upd_stamp || ctx->upd_call == 0xffffffffu) {
    CK(ctx->d_upd_stamp.reserve(ctx->V));
    CK(cudaMemsetAsync(ctx->d_upd_stamp, 0, sizeof(uint32_t) * (size_t)ctx->V, ctx->stream));
    ctx->upd_call = 0;
  }
  ++ctx->upd_call;
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  unsigned launches = 1;
  MNB_LAUNCH(k_update_costs, (n_changed + 255) / 256, 256, 0, ctx->stream, d_ids, n_changed, d_costs, (int)(costs_indexed_by_vertex != 0),
             default_value, ctx->V, ctx->d_cost, ctx->d_upd_stamp, ctx->upd_call);
  if (edge_cost_factor != 0) {                       // mesh_map.cpp:568-572: no edge update at all for a zero factor
    const unsigned blocks = (unsigned)(((size_t)n_changed * ELL_W + 255) / 256);
    MNB_LAUNCH(k_update_edge_weights, blocks, 256, 0, ctx->stream, d_ids, n_changed, ctx->V, (const uint32_t*)ctx->d_adj_ptr,
               (const uint32_t*)ctx->d_adj_eid, (const uint32_t*)ctx->d_edges, (const float*)ctx->d_cost, (const float*)ctx->d_edge_dist,
               edge_cost_factor, ctx->d_edge_w);
    RefreshArgs r{};
    r.changed = d_ids; r.n = n_changed; r.V = ctx->V; r.faces = ctx->d_faces; r.cor_ptr = ctx->d_cor_ptr; r.cor_idx = ctx->d_cor_idx;
    r.cor_eid = ctx->d_cor_eid; r.face_cor = ctx->d_face_cor; r.adj_ptr = ctx->d_adj_ptr; r.adj_nbr = ctx->d_adj_nbr; r.adj_eid = ctx->d_adj_eid; r.w = ctx->d_edge_w;
    r.cor_w = ctx->d_cor_w; r.ell_w = ctx->d_ell_w; r.ell_geo = ctx->d_ell_geo;
    r.adj_nw = ctx->adj_dirty ? nullptr : ctx->d_adj_nw.p; r.ell_adj = ctx->adj_dirty ? nullptr : ctx->d_ell_adj.p;   // stale tables are rebuilt whole anyway
    r.stamp = ctx->d_upd_stamp; r.call = ctx->upd_call;
    MNB_LAUNCH(k_refresh_weight_tables, blocks, 256, 0, ctx->stream, r);
    launches = 3;
  }
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  simple_stats(ctx, launches, n_changed);
  return MNB_OK;
}

}  // extern "C"

static int32_t combination_update(mnb_ctx* ctx, uint32_t n_layers, const float* const* layer_costs, const float* defaults,
                                  const float* weights /* null: MaxCombinationLayer */, const uint8_t* const* layer_lethal,
                                  uint32_t n_changed, const uint32_t* changed, float* io_costs, uint8_t* io_lethal) {
  if (!ctx || !ctx->V || n_layers == 0 || n_layers > (uint32_t)COMB_MAX_LAYERS || !layer_costs || !defaults || !io_costs ||
      (n_changed && !changed)) return MNB_E_ARG;
  for (uint32_t l = 0; l < n_layers; ++l) if (!layer_costs[l]) return MNB_E_ARG;
  if (n_changed == 0) return MNB_OK;
  CK(cudaSetDevice(ctx->device));
  const size_t V = ctx->V;
  CombineArgs a{};
  a.n_layers = n_layers; a.n = n_changed; a.V = ctx->V; a.average = weights ? 1 : 0;
  for (uint32_t l = 0; l < n_layers; ++l) a.weight[l] = weights ? weights[l] : 1.0f;
  // host-pointer mode: device copies of the maps, for this call
  DeviceBuffer<float> d_costs[COMB_MAX_LAYERS], d_io; DeviceBuffer<uint8_t> d_lethal[COMB_MAX_LAYERS], d_il; DeviceBuffer<uint32_t> d_ids;
  CallerArrays io(ctx);
  for (uint32_t l = 0; l < n_layers; ++l) {
    a.def[l] = defaults[l];
    a.costs[l] = io.in(layer_costs[l], d_costs[l], V);
    a.lethal[l] = layer_lethal ? io.in(layer_lethal[l], d_lethal[l], V) : nullptr;
  }
  a.changed = io.in(changed, d_ids, n_changed);
  a.io_costs = io.inout(io_costs, d_io, V);
  a.io_lethal = io.inout(io_lethal, d_il, V);
  CK(io.status());
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  MNB_LAUNCH(k_max_combination_update, (n_changed + 255) / 256, 256, 0, ctx->stream, a);
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(io.copy_back());
  CK(cudaStreamSynchronize(ctx->stream));
  simple_stats(ctx, 1, n_changed);
  return MNB_OK;
}

extern "C" {

static int32_t impl_max_combination_update(mnb_ctx* ctx, uint32_t n_layers, const float* const* layer_costs, const float* defaults,
                                   const uint8_t* const* layer_lethal, uint32_t n_changed, const uint32_t* changed,
                                   float* io_costs, uint8_t* io_lethal) {
  return combination_update(ctx, n_layers, layer_costs, defaults, nullptr, layer_lethal, n_changed, changed, io_costs, io_lethal);
}

static int32_t impl_avg_combination_update(mnb_ctx* ctx, uint32_t n_layers, const float* const* layer_costs, const float* defaults,
                                   const float* weights, const uint8_t* const* layer_lethal, uint32_t n_changed,
                                   const uint32_t* changed, float* io_costs, uint8_t* io_lethal) {
  if (!weights) return MNB_E_ARG;
  return combination_update(ctx, n_layers, layer_costs, defaults, weights, layer_lethal, n_changed, changed, io_costs, io_lethal);
}

// ---- exception barrier: nothing propagates through the C ABI; a failed call leaves no half-built state behind ----
int32_t mnb_set_mesh(mnb_ctx* ctx, uint32_t V, uint32_t F, const float* pos, const uint32_t* faces,
                     const uint32_t* edges, uint32_t E) {
  const int32_t rc = guarded(ctx, [&]() { return impl_set_mesh(ctx, V, F, pos, faces, edges, E); });
  if (rc != MNB_OK && ctx) free_mesh(ctx);      // no half-built context (V = F = E = 0)
  return rc;
}
int32_t mnb_cvp(mnb_ctx* ctx, uint32_t seed_face, const float seed_pos[3], int64_t robot_face, double cost_limit,
                double goal_dist_offset, float* out_dist, uint32_t* out_pred, float* out_direction, int32_t* out_cut) {
  return guarded(ctx, [&]() { return impl_cvp(ctx, seed_face, seed_pos, robot_face, cost_limit, goal_dist_offset, out_dist, out_pred, out_direction, out_cut); });
}
int32_t mnb_cvp_replan(mnb_ctx* ctx, uint32_t seed_face, const float seed_pos[3], int64_t robot_face, double cost_limit,
                       double goal_dist_offset, uint32_t n_changed, const uint32_t* changed, float* out_dist, uint32_t* out_pred,
                       float* out_direction, int32_t* out_cut) {
  return guarded(ctx, [&]() { return impl_cvp_replan(ctx, seed_face, seed_pos, robot_face, cost_limit, goal_dist_offset, n_changed, changed,
                                                     out_dist, out_pred, out_direction, out_cut); });
}
int32_t mnb_cvp_batch_fields(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_faces, const float* seed_pos, double cost_limit,
                             float* out_dist, uint32_t* out_pred, float* out_direction, int32_t* out_cutting_face) {
  return guarded(ctx, [&]() {
    return impl_cvp_batch_fields(ctx, n, seed_faces, seed_pos, cost_limit, out_dist, out_pred, out_direction, out_cutting_face);
  });
}
int32_t mnb_cvp_batch_replan(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_faces, const float* seed_pos, double cost_limit,
                             uint32_t n_changed, const uint32_t* changed, float* out_dist, uint32_t* out_pred, float* out_direction,
                             int32_t* out_cutting_face) {
  return guarded(ctx, [&]() {
    return impl_cvp_batch_replan(ctx, n, seed_faces, seed_pos, cost_limit, n_changed, changed, out_dist, out_pred, out_direction, out_cutting_face);
  });
}
int32_t mnb_cvp_batch_replan_release(mnb_ctx* ctx) {
  if (!ctx) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  ctx->brs.clear();
  return MNB_OK;
}
int32_t mnb_cvp_batch(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_faces, const float* seed_pos, double cost_limit,
                      float* out_dist) {
  return guarded(ctx, [&]() { return impl_cvp_batch_fields(ctx, n, seed_faces, seed_pos, cost_limit, out_dist, nullptr, nullptr, nullptr); });
}
int32_t mnb_dijkstra(mnb_ctx* ctx, uint32_t seed_vertex, int64_t robot_vertex, double cost_limit, double goal_dist_offset,
                     float* out_dist, uint32_t* out_pred) {
  return guarded(ctx, [&]() { return impl_dijkstra(ctx, seed_vertex, robot_vertex, cost_limit, goal_dist_offset, out_dist, out_pred); });
}
int32_t mnb_dijkstra_batch(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_vertices, double cost_limit, float* out_dist,
                           uint32_t* out_pred) {
  return guarded(ctx, [&]() { return impl_dijkstra_batch(ctx, n, seed_vertices, cost_limit, out_dist, out_pred); });
}
int32_t mnb_dijkstra_batch_repair(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_vertices, double cost_limit, uint32_t n_changed,
                                  const uint32_t* changed, float* io_dist, uint32_t* io_pred) {
  const RepairRequest rq{n_changed, changed};
  return guarded(ctx, [&]() { return impl_dijkstra_batch(ctx, n, seed_vertices, cost_limit, io_dist, io_pred, nullptr, &rq); });
}
int32_t mnb_dijkstra_matrix(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_vertices, uint32_t m, const uint32_t* target_vertices,
                            double cost_limit, float* out) {
  if (!ctx || m == 0 || !target_vertices || !out) return MNB_E_ARG;
  const MatrixRequest mx{m, target_vertices, out};
  return guarded(ctx, [&]() { return impl_dijkstra_batch(ctx, n, seed_vertices, cost_limit, nullptr, nullptr, &mx); });
}
int32_t mnb_cvp_matrix(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_faces, const float* seed_pos, uint32_t m,
                       const uint32_t* target_vertices, double cost_limit, float* out) {
  if (!ctx || m == 0 || !target_vertices || !out) return MNB_E_ARG;
  const MatrixRequest mx{m, target_vertices, out};
  return guarded(ctx, [&]() { return impl_cvp_batch_fields(ctx, n, seed_faces, seed_pos, cost_limit, nullptr, nullptr, nullptr, nullptr, &mx); });
}
int32_t mnb_inflate(mnb_ctx* ctx, const uint32_t* lethals, uint32_t n, const uint8_t* invalid,
                    const mnb_inflation_params* params, float* out_dist, float* out_cost) {
  return guarded(ctx, [&]() { return impl_inflate(ctx, lethals, n, invalid, params, out_dist, out_cost); });
}
int32_t mnb_inflation_update(mnb_ctx* ctx, const uint32_t* lethals, uint32_t n, const uint8_t* invalid,
                             const mnb_inflation_params* params, float* out_dist, float* out_cost, uint32_t* out_changed,
                             uint32_t* n_changed) {
  return guarded(ctx, [&]() { return impl_inflation_update(ctx, lethals, n, invalid, params, out_dist, out_cost, out_changed, n_changed); });
}
int32_t mnb_compute_layers(mnb_ctx* ctx, const mnb_layer_params* params, const float* clearance, float* out_costs,
                           float* out_combined, uint8_t* out_lethal_mask) {
  return guarded(ctx, [&]() { return impl_compute_layers(ctx, params, clearance, out_costs, out_combined, out_lethal_mask); });
}
int32_t mnb_set_costs(mnb_ctx* ctx, const float* vertex_costs, const float* edge_weights, const uint8_t* invalid) {
  return guarded(ctx, [&]() { return impl_set_costs(ctx, vertex_costs, edge_weights, invalid); });
}
int32_t mnb_compute_edge_weights(mnb_ctx* ctx, const float* vertex_costs, double edge_cost_factor, float* out_w) {
  return guarded(ctx, [&]() { return impl_compute_edge_weights(ctx, vertex_costs, edge_cost_factor, out_w); });
}
int32_t mnb_locate(mnb_ctx* ctx, uint32_t n, const float* points, uint32_t* out_vertex, int32_t* out_face, float* out_bary) {
  return guarded(ctx, [&]() { return impl_locate(ctx, n, points, out_vertex, out_face, out_bary); });
}
int32_t mnb_vector_map(mnb_ctx* ctx, const uint32_t* pred, const float* direction, const int32_t* cutting_face, float* out_vec) {
  return guarded(ctx, [&]() { return impl_vector_map(ctx, pred, direction, cutting_face, out_vec); });
}
int32_t mnb_inflation_repair(mnb_ctx* ctx, const uint32_t* lethals, uint32_t n, const uint8_t* invalid,
                             const mnb_inflation_params* params, float* out_dist, float* out_cost, uint32_t* out_changed,
                             uint32_t* n_changed) {
  return guarded(ctx, [&]() { return impl_inflation_repair(ctx, lethals, n, invalid, params, out_dist, out_cost, out_changed, n_changed); });
}
int32_t mnb_inflation_vector_map(mnb_ctx* ctx, float* out_vectors) {
  return guarded(ctx, [&]() { return impl_inflation_vector_map(ctx, out_vectors); });
}
int32_t mnb_inflation_vector_at(mnb_ctx* ctx, uint32_t n, const uint32_t* faces_q, const float* bary, float* out) {
  return guarded(ctx, [&]() { return impl_inflation_vector_at(ctx, n, faces_q, bary, out); });
}
int32_t mnb_cvp_backtrack(mnb_ctx* ctx, const float robot_pos[3], uint32_t robot_face, double step_width, uint32_t max_points,
                          float* path_pos, uint32_t* path_face, uint32_t* n_points) {
  return guarded(ctx, [&]() { return impl_cvp_backtrack(ctx, robot_pos, robot_face, step_width, max_points, path_pos, path_face, n_points); });
}
int32_t mnb_update_vertex_costs(mnb_ctx* ctx, uint32_t n_changed, const uint32_t* changed, const float* costs,
                                int32_t costs_indexed_by_vertex, float default_value, double edge_cost_factor) {
  return guarded(ctx, [&]() { return impl_update_vertex_costs(ctx, n_changed, changed, costs, costs_indexed_by_vertex, default_value, edge_cost_factor); });
}
int32_t mnb_max_combination_update(mnb_ctx* ctx, uint32_t n_layers, const float* const* layer_costs, const float* defaults,
                                   const uint8_t* const* layer_lethal, uint32_t n_changed, const uint32_t* changed,
                                   float* io_costs, uint8_t* io_lethal) {
  return guarded(ctx, [&]() { return impl_max_combination_update(ctx, n_layers, layer_costs, defaults, layer_lethal, n_changed, changed, io_costs, io_lethal); });
}
int32_t mnb_avg_combination_update(mnb_ctx* ctx, uint32_t n_layers, const float* const* layer_costs, const float* defaults,
                                   const float* weights, const uint8_t* const* layer_lethal, uint32_t n_changed,
                                   const uint32_t* changed, float* io_costs, uint8_t* io_lethal) {
  return guarded(ctx, [&]() { return impl_avg_combination_update(ctx, n_layers, layer_costs, defaults, weights, layer_lethal, n_changed, changed, io_costs, io_lethal); });
}

}  // extern "C"

#include "raycast_host.cuh"
#include "group.cuh"
