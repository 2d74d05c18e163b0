// Planner vector maps, the inflation wave + its repulsive vector field, vector-field back-tracking, localisation.
// (part of libmeshnav_b200.so: included by meshnav.cu, which holds the C ABI and all host code)
#pragma once
#include "launch.cuh"
#include "kernels_wavefront.cuh"

using namespace mnb;

// ============================================================================
// Vector-field epilogues: DijkstraMeshPlanner::computeVectorMap (dijkstra_mesh_planner.cpp:189-209) and
// CVPMeshPlanner::computeVectorMap (cvp_mesh_planner.cpp:204-239).  NaN = "no entry in the sparse map".
// ============================================================================
struct F3 { float x, y, z; };
__device__ __forceinline__ F3 f3sub(F3 a, F3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ F3 f3cross(F3 a, F3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
__device__ __forceinline__ float f3dot(F3 a, F3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ F3 f3load(const float* __restrict__ p, uint32_t v) { return {p[3 * (size_t)v], p[3 * (size_t)v + 1], p[3 * (size_t)v + 2]}; }
__device__ __forceinline__ F3 f3normalized(F3 v) {
  const float l = sqrtf(v.x * v.x + v.y * v.y + v.z * v.z);
  if (l > 0) { v.x /= l; v.y /= l; v.z /= l; }
  return v;
}

// one entry of the planners' vector map; false = "no entry" (pred == self or no cutting face)
__device__ __forceinline__ bool vertex_vector(const float* __restrict__ pos, const float* __restrict__ vn,
                                              const uint32_t* __restrict__ pred, const float* __restrict__ direction,
                                              const int32_t* __restrict__ cut, uint32_t v3, F3& out) {
  const uint32_t v1 = pred[v3];
  if (v1 == v3 || (cut && cut[v3] < 0)) return false;
  F3 v = f3sub(f3load(pos, v1), f3load(pos, v3));
  if (direction) {   // rotate about the vertex normal by the stored angle (Rodrigues; lvr2 BaseVector::rotated)
    const F3 n = f3load(vn, v3);
    const double alpha = (double)direction[v3];
    const float sina = (float)sin(alpha), cosa = (float)cos(alpha);
    const float ndotv = f3dot(n, v);
    const F3 c = f3cross(n, v);
    v = {v.x * cosa + c.x * sina + n.x * ndotv * (1.0f - cosa), v.y * cosa + c.y * sina + n.y * ndotv * (1.0f - cosa),
         v.z * cosa + c.z * sina + n.z * ndotv * (1.0f - cosa)};
  }
  out = f3normalized(v);
  return true;
}

__global__ void k_vector_map(const float* __restrict__ pos, const float* __restrict__ vn, const uint32_t* __restrict__ pred,
                             const float* __restrict__ direction, const int32_t* __restrict__ cut, uint32_t V,
                             float* __restrict__ out) {
  const uint32_t v3 = blockIdx.x * blockDim.x + threadIdx.x;
  if (v3 >= V) return;
  const float nan = __int_as_float(0x7fc00000);
  F3 v{nan, nan, nan};
  vertex_vector(pos, vn, pred, direction, cut, v3, v);
  float* o = out + 3 * (size_t)v3;
  o[0] = v.x; o[1] = v.y; o[2] = v.z;
}

// ============================================================================
// InflationLayer::waveCostInflation (inflation_layer.cpp:341-491): whole-grid cooperative kernel
// (multi-source: few, very wide rounds) + fading epilogue (:482-490, :315-339)
// ============================================================================
struct InflateKernelArgs {
  uint32_t V;
  const uint32_t* cor_ptr; const int4* cor_idx; const float4* cor_wd; const uint4* cor_eid;
  const uint8_t* invalid;
  WaveWorkspace ws;
  const uint32_t* lethals; uint32_t n_lethals;
  float max_distance;
  InflationParams params;
  float* out_dist; float* out_cost;
  uint32_t max_rounds;
  int skip_clean;
};

#ifndef MNB_INFL_MINBLOCKS
#define MNB_INFL_MINBLOCKS 1
#endif
__global__ void __launch_bounds__(512, MNB_INFL_MINBLOCKS) k_inflate(const InflateKernelArgs a) {
  __shared__ Stage st;
  uint32_t g, gthreads, gtid;
  group_coords<0>(g, gthreads, gtid);
  const uint32_t V = a.V;
  uint4* state = a.ws.state; uint32_t* mark = a.ws.mark; uint32_t* list0 = a.ws.list0; uint32_t* list1 = a.ws.list1;
  GroupCtl* ctl = a.ws.ctl;
  if (threadIdx.x == 0) { st.n = 0; st.m_tau = INF_BITS; st.lo = INF_BITS; }
  __syncthreads();
#pragma unroll 4
  for (uint32_t v = gtid; v < V; v += gthreads) { state[v] = state_inf(); mark[v] = MARK_NONE; a.ws.chg[v] = 0u; a.ws.last_eval[v] = 0u; a.ws.dirty[v] = 0u; }
  group_sync<0>(ctl->barrier);
  for (uint32_t i = gtid; i < a.n_lethals; i += gthreads) {      // :397-402
    const uint32_t v = a.lethals[i];
    if (v < V) { state[v] = make_uint4(0u, 0u, 0u, 0u); mark[v] = MARK_FIXED; }
  }
  if (gtid == 0) ctl_reset(ctl, 0, 0.0f);
  group_sync<0>(ctl->barrier);
  InflationProblem prob;
  prob.cor_ptr = a.cor_ptr; prob.cor_idx = a.cor_idx; prob.cor_wd = a.cor_wd; prob.cor_eid = a.cor_eid; prob.invalid = a.invalid;
  prob.state = state; prob.ext_arr = a.ws.ext; prob.root_arr = a.ws.root; prob.chg = a.ws.chg;
  prob.pool_w = a.ws.pool; prob.pool = prob.pool_w; prob.pool_cap = a.ws.pool_cap; prob.pool_top = &ctl->pool_top; prob.pool_overflow = &ctl->pool_overflow;
  prob.deferred_m = __uint_as_float(INF_BITS); prob.max_distance = a.max_distance;
  prob.last_eval = a.ws.last_eval; prob.dirty_round = a.ws.dirty; prob.skip_clean = a.skip_clean; prob.deferred_flag = false;
  for (uint32_t i = gtid; i < a.n_lethals; i += gthreads) {
    const uint32_t v = a.lethals[i];
    if (v >= V) continue;
    prob.activate(v, [&](uint32_t x) {
      if (__ldcg(&mark[x]) == MARK_NONE && atomicCAS(&mark[x], MARK_NONE, MARK_CAND) == MARK_NONE)
        stage_push(st, x, list0, &ctl->count[0]);
    });
  }
  stage_flush(st, list0, &ctl->count[0], &ctl->m_tau[0], &ctl->lo[0]);
  group_sync<0>(ctl->barrier);
  run_band_rounds<0>(prob, ctl, list0, list1, mark, st, __uint_as_float(INF_BITS), gthreads, gtid, 0, 0u, 0u, 0u, 0.0,
                     nullptr, 1e-30f, a.max_rounds);
  group_sync<0>(ctl->barrier);
  // dense outputs: four independent label loads in flight per thread (the loop is a stream over V, not part of the wave)
  for (uint32_t v0 = gtid; v0 < V; v0 += 4 * gthreads) {
    float d[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) { const uint32_t v = v0 + q * gthreads; d[q] = v < V ? __uint_as_float(__ldcg(reinterpret_cast<const uint32_t*>(state) + 4 * (size_t)v)) : 0.0f; }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t v = v0 + q * gthreads;
      if (v >= V) continue;
      if (a.out_dist) a.out_dist[v] = d[q];
      if (a.out_cost) a.out_cost[v] = (__float_as_uint(d[q]) == INF_BITS) ? __int_as_float(0x7fc00000) : fading(a.params, d[q]);
    }
  }
}

// ============================================================================
// InflationLayer repulsive vector field, vector_map_ (inflation_layer.cpp:277-308), from the final labels of k_inflate.
// The reference accumulates it inside the sequential loop; the result factors into two phases (oracle: orc_inflation):
//  (1) while the lethal vertices pop (all at key 0, in id order) every face with exactly two lethal vertices adds its
//      direction to the vectors of its three vertices, once per (popping vertex, incident edge of the face, side of the
//      edge) -- `vec = (vec + dir).normalized()` in exactly that order (:277-295).  Per vertex this is an ordered fold over
//      at most 4 events per incident face: gathered, sorted by (popping vertex, edge position, side) and folded here.
//  (2) afterwards a vertex' vector is overwritten by every accepted update with a non-lethal source,
//      (vec[v1]*(u3-u1) + vec[v2]*(u3-u2)).normalized() (:301-308): the LAST accepted face of the event-ordered replay
//      decides; its sources popped earlier, so their vectors are final -- evaluated by fixed-point iteration over the
//      (acyclic) source relation.
// ============================================================================
struct InflVecArgs {
  uint32_t V;
  const float* pos; const uint32_t* faces;
  const uint32_t* cor_ptr; const int4* cor_idx; const float4* cor_wd; const uint4* cor_eid;
  const uint32_t* adj_ptr; const uint32_t* adj_nbr;
  const uint8_t* invalid;
  WaveWorkspace ws;
  float max_distance;
  float* vec;                  // 3V, zero = no entry
  int4* src;                   // {v1, v2, bits(u3-u1), bits(u3-u2)}; v1 = -1: no overwrite
  unsigned int* flag;          // [0] a vector changed in this sweep, [1] scratch overflow
};
constexpr int IV_MAXF = 24, IV_MAXE = 4 * IV_MAXF;

__device__ __forceinline__ float iv_len(const float* __restrict__ pos, uint32_t p, uint32_t q) {   // == k_edge_dist
  const float dx = pos[3 * (size_t)p] - pos[3 * (size_t)q], dy = pos[3 * (size_t)p + 1] - pos[3 * (size_t)q + 1],
              dz = pos[3 * (size_t)p + 2] - pos[3 * (size_t)q + 2];
  return sqrtf(dx * dx + dy * dy + dz * dz);
}

// The per-vertex bodies of the three kernels, shared with the repair's vertex-list kernels (kernels_infl_repair.cuh).
// k_infl_vec_lethal keeps its own copy of the first: calling the shared body costs it one register.
__device__ __forceinline__ void infl_vec_lethal_at(const InflVecArgs a, uint32_t x) {
  if (x >= a.V) return;
  float* out = a.vec + 3 * (size_t)x;
  out[0] = 0.0f; out[1] = 0.0f; out[2] = 0.0f;
  unsigned long long key[IV_MAXE]; uint8_t ev_face[IV_MAXE];
  F3 fdir[IV_MAXF];
  int ne = 0, nf = 0;
  for (uint32_t k = a.cor_ptr[x]; k < a.cor_ptr[x + 1]; ++k) {
    const uint32_t f = (uint32_t)a.cor_idx[k].z;
    const uint32_t fa = a.faces[3 * (size_t)f], fb = a.faces[3 * (size_t)f + 1], fc = a.faces[3 * (size_t)f + 2];
    const bool la = __uint_as_float(a.ws.state[fa].x) == 0.0f, lb = __uint_as_float(a.ws.state[fb].x) == 0.0f,
               lc = __uint_as_float(a.ws.state[fc].x) == 0.0f;
    uint32_t w1, w2, w3;                                       // argument order of waveFrontUpdate (:445-470)
    if (la && lb && !lc) { w1 = fa; w2 = fb; w3 = fc; }
    else if (la && !lb && lc) { w1 = fc; w2 = fa; w3 = fb; }
    else if (!la && lb && lc) { w1 = fb; w2 = fc; w3 = fa; }
    else continue;
    const float cand = inflation_candidate(0.0f, 0.0f, iv_len(a.pos, w2, w3), iv_len(a.pos, w1, w3), iv_len(a.pos, w1, w2));
    if (__float_as_uint(cand) == INF_BITS) continue;           // :271 non-finite update: the call returns before the vectors
    if (nf >= IV_MAXF) { atomicAdd(&a.flag[1], 1u); return; }
    const F3 p1 = f3load(a.pos, w1), p2 = f3load(a.pos, w2), p3 = f3load(a.pos, w3);
    fdir[nf] = f3normalized(F3{(p3.x - p2.x) + (p3.x - p1.x), (p3.y - p2.y) + (p3.y - p1.y), (p3.z - p2.z) + (p3.z - p1.z)});
    const uint32_t lv[2] = {w1, w2};
    for (int s = 0; s < 2; ++s) {
      const uint32_t p = lv[s];                                // the popping lethal vertex
      if (a.invalid && a.invalid[p]) continue;                 // pops but does not expand (:417)
      const uint32_t others[2] = {p == w1 ? w2 : w1, w3};
      for (int t = 0; t < 2; ++t) {
        const uint32_t q = others[t];
        uint32_t epos = 0;                                     // position of edge (p,q) among p's edges (ascending edge id)
        for (uint32_t kk = a.adj_ptr[p]; kk < a.adj_ptr[p + 1]; ++kk) if (a.adj_nbr[kk] == q) { epos = kk - a.adj_ptr[p]; break; }
        uint32_t side = 0;                                     // an edge lists its faces in ascending id
        for (uint32_t kk = a.cor_ptr[p]; kk < a.cor_ptr[p + 1]; ++kk) {
          const int4 ix = a.cor_idx[kk];
          if ((uint32_t)ix.z != f && ((uint32_t)ix.x == q || (uint32_t)ix.y == q)) { side = (uint32_t)ix.z < f ? 1u : 0u; break; }
        }
        key[ne] = ((unsigned long long)p << 32) | ((unsigned long long)epos << 1) | side;
        ev_face[ne] = (uint8_t)nf; ++ne;
      }
    }
    ++nf;
  }
  if (ne == 0) return;
  F3 v{0.0f, 0.0f, 0.0f};
  for (int i = 0; i < ne; ++i) {                               // selection sort: <= 96 events, usually 4-16
    int b = i;
    for (int j = i + 1; j < ne; ++j) if (key[j] < key[b]) b = j;
    const unsigned long long kb = key[b]; const uint8_t fbi = ev_face[b];
    key[b] = key[i]; ev_face[b] = ev_face[i]; key[i] = kb; ev_face[i] = fbi;
    const F3 d = fdir[fbi];
    v = f3normalized(F3{v.x + d.x, v.y + d.y, v.z + d.z});
  }
  out[0] = v.x; out[1] = v.y; out[2] = v.z;
}
__global__ void __launch_bounds__(128) k_infl_vec_lethal(const InflVecArgs a) {
  const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= a.V) return;
  float* out = a.vec + 3 * (size_t)x;
  out[0] = 0.0f; out[1] = 0.0f; out[2] = 0.0f;
  unsigned long long key[IV_MAXE]; uint8_t ev_face[IV_MAXE];
  F3 fdir[IV_MAXF];
  int ne = 0, nf = 0;
  for (uint32_t k = a.cor_ptr[x]; k < a.cor_ptr[x + 1]; ++k) {
    const uint32_t f = (uint32_t)a.cor_idx[k].z;
    const uint32_t fa = a.faces[3 * (size_t)f], fb = a.faces[3 * (size_t)f + 1], fc = a.faces[3 * (size_t)f + 2];
    const bool la = __uint_as_float(a.ws.state[fa].x) == 0.0f, lb = __uint_as_float(a.ws.state[fb].x) == 0.0f,
               lc = __uint_as_float(a.ws.state[fc].x) == 0.0f;
    uint32_t w1, w2, w3;                                       // argument order of waveFrontUpdate (:445-470)
    if (la && lb && !lc) { w1 = fa; w2 = fb; w3 = fc; }
    else if (la && !lb && lc) { w1 = fc; w2 = fa; w3 = fb; }
    else if (!la && lb && lc) { w1 = fb; w2 = fc; w3 = fa; }
    else continue;
    const float cand = inflation_candidate(0.0f, 0.0f, iv_len(a.pos, w2, w3), iv_len(a.pos, w1, w3), iv_len(a.pos, w1, w2));
    if (__float_as_uint(cand) == INF_BITS) continue;           // :271 non-finite update: the call returns before the vectors
    if (nf >= IV_MAXF) { atomicAdd(&a.flag[1], 1u); return; }
    const F3 p1 = f3load(a.pos, w1), p2 = f3load(a.pos, w2), p3 = f3load(a.pos, w3);
    fdir[nf] = f3normalized(F3{(p3.x - p2.x) + (p3.x - p1.x), (p3.y - p2.y) + (p3.y - p1.y), (p3.z - p2.z) + (p3.z - p1.z)});
    const uint32_t lv[2] = {w1, w2};
    for (int s = 0; s < 2; ++s) {
      const uint32_t p = lv[s];                                // the popping lethal vertex
      if (a.invalid && a.invalid[p]) continue;                 // pops but does not expand (:417)
      const uint32_t others[2] = {p == w1 ? w2 : w1, w3};
      for (int t = 0; t < 2; ++t) {
        const uint32_t q = others[t];
        uint32_t epos = 0;                                     // position of edge (p,q) among p's edges (ascending edge id)
        for (uint32_t kk = a.adj_ptr[p]; kk < a.adj_ptr[p + 1]; ++kk) if (a.adj_nbr[kk] == q) { epos = kk - a.adj_ptr[p]; break; }
        uint32_t side = 0;                                     // an edge lists its faces in ascending id
        for (uint32_t kk = a.cor_ptr[p]; kk < a.cor_ptr[p + 1]; ++kk) {
          const int4 ix = a.cor_idx[kk];
          if ((uint32_t)ix.z != f && ((uint32_t)ix.x == q || (uint32_t)ix.y == q)) { side = (uint32_t)ix.z < f ? 1u : 0u; break; }
        }
        key[ne] = ((unsigned long long)p << 32) | ((unsigned long long)epos << 1) | side;
        ev_face[ne] = (uint8_t)nf; ++ne;
      }
    }
    ++nf;
  }
  if (ne == 0) return;
  F3 v{0.0f, 0.0f, 0.0f};
  for (int i = 0; i < ne; ++i) {                               // selection sort: <= 96 events, usually 4-16
    int b = i;
    for (int j = i + 1; j < ne; ++j) if (key[j] < key[b]) b = j;
    const unsigned long long kb = key[b]; const uint8_t fbi = ev_face[b];
    key[b] = key[i]; ev_face[b] = ev_face[i]; key[i] = kb; ev_face[i] = fbi;
    const F3 d = fdir[fbi];
    v = f3normalized(F3{v.x + d.x, v.y + d.y, v.z + d.z});
  }
  out[0] = v.x; out[1] = v.y; out[2] = v.z;
}

__device__ __forceinline__ void infl_vec_sources_at(const InflVecArgs& a, uint32_t c) {
  if (c >= a.V) return;
  int4 r = make_int4(-1, -1, 0, 0);
  const float d = __uint_as_float(a.ws.state[c].x);
  if (d != 0.0f && __float_as_uint(d) != INF_BITS) {
    InflationProblem prob;
    prob.cor_ptr = a.cor_ptr; prob.cor_idx = a.cor_idx; prob.cor_wd = a.cor_wd; prob.cor_eid = a.cor_eid; prob.invalid = a.invalid;
    prob.state = a.ws.state; prob.ext_arr = a.ws.ext; prob.root_arr = a.ws.root; prob.chg = a.ws.chg;
    prob.pool_w = a.ws.pool; prob.pool = prob.pool_w; prob.pool_cap = a.ws.pool_cap; prob.pool_top = &a.ws.ctl->pool_top; prob.pool_overflow = &a.ws.ctl->pool_overflow;
    prob.deferred_m = __uint_as_float(INF_BITS); prob.strict = 0; prob.max_distance = a.max_distance;
    prob.last_eval = nullptr; prob.dirty_round = nullptr; prob.skip_clean = 0; prob.deferred_flag = false;
    float nd, wu1, wu2; EvFull tc; int win;
    prob.replay(c, __uint_as_float(INF_BITS), 0xfffffff0u /* final labels: nothing is deferred */, nd, tc, win, wu1, wu2);
    if (win >= 0 && (wu1 != 0.0f || wu2 != 0.0f)) {           // :301 (an update from two lethal sources keeps the phase-1 vector)
      const int4 ix = a.cor_idx[win];
      r = make_int4(ix.x, ix.y, __float_as_int(nd - wu1), __float_as_int(nd - wu2));
    }
  }
  a.src[c] = r;
}
__global__ void __launch_bounds__(128) k_infl_vec_sources(const InflVecArgs a) {
  infl_vec_sources_at(a, blockIdx.x * blockDim.x + threadIdx.x);
}

__device__ __forceinline__ void infl_vec_sweep_at(const InflVecArgs a, uint32_t c) {
  const int4 r = a.src[c];
  if (r.x < 0) return;
  const float d31 = __int_as_float(r.z), d32 = __int_as_float(r.w);
  const float* va = a.vec + 3 * (size_t)r.x; const float* vb = a.vec + 3 * (size_t)r.y;
  const F3 v = f3normalized(F3{va[0] * d31 + vb[0] * d32, va[1] * d31 + vb[1] * d32, va[2] * d31 + vb[2] * d32});   // :306
  float* out = a.vec + 3 * (size_t)c;
  if (__float_as_uint(out[0]) != __float_as_uint(v.x) || __float_as_uint(out[1]) != __float_as_uint(v.y) ||
      __float_as_uint(out[2]) != __float_as_uint(v.z)) {
    out[0] = v.x; out[1] = v.y; out[2] = v.z;
    a.flag[0] = 1u;
  }
}
__global__ void __launch_bounds__(256) k_infl_vec_sweep(const InflVecArgs a) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.V) return;
  infl_vec_sweep_at(a, c);
}

// InflationLayer::vectorAt(vertices, barycentric_coords) (inflation_layer.cpp:493-521); see oracle inflationVectorAt
struct RepulsiveField {
  const float* dist; const float* vec;   // null = no repulsive layer
  float inscribed_radius_f; double inscribed_radius, inflation_radius; float lethal_value, inscribed_value;
};
__device__ __forceinline__ F3 inflation_vector_at(const RepulsiveField& L, const uint32_t* __restrict__ t, const float bary[3]) {
  const float d0 = L.dist[t[0]], d1 = L.dist[t[1]], d2 = L.dist[t[2]];
  if (!isfinite(d0) || !isfinite(d1) || !isfinite(d2)) return F3{0.0f, 0.0f, 0.0f};
  const float distance = d0 * bary[0] + d1 * bary[1] + d2 * bary[2];
  if ((double)distance > L.inflation_radius) return F3{0.0f, 0.0f, 0.0f};
  const F3 va = f3load(L.vec, t[0]), vb = f3load(L.vec, t[1]), vc = f3load(L.vec, t[2]);
  const F3 v{va.x * bary[0] + vb.x * bary[1] + vc.x * bary[2], va.y * bary[0] + vb.y * bary[1] + vc.y * bary[2],
             va.z * bary[0] + vb.z * bary[1] + vc.z * bary[2]};
  if ((double)distance > L.inscribed_radius) {
    const float alpha = (float)(((double)sqrtf(distance) - L.inscribed_radius) / (L.inflation_radius - L.inscribed_radius) * 3.14159265358979323846);
    const float s1 = L.inscribed_value, s2 = cosf(alpha) + 1, s3 = 2.0f;
    return F3{v.x * s1 * s2 / s3, v.y * s1 * s2 / s3, v.z * s1 * s2 / s3};
  }
  const float s = distance > 0 ? L.inscribed_value : L.lethal_value;
  return F3{v.x * s, v.y * s, v.z * s};
}
__global__ void k_inflation_vector_at(const RepulsiveField L, const uint32_t* __restrict__ faces, uint32_t n,
                                      const uint32_t* __restrict__ faces_q, const float* __restrict__ bary, float* __restrict__ out) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const float b[3] = {bary[3 * (size_t)q], bary[3 * (size_t)q + 1], bary[3 * (size_t)q + 2]};
  const F3 v = inflation_vector_at(L, faces + 3 * (size_t)faces_q[q], b);
  out[3 * (size_t)q] = v.x; out[3 * (size_t)q + 1] = v.y; out[3 * (size_t)q + 2] = v.z;
}

// ============================================================================
// Vector-field back-tracking (cvp_mesh_planner.cpp:920-951): MeshMap::meshAhead (mesh_map.cpp:1070-1108),
// searchNeighbourFaces (:999-1068), directionAtPosition (:625-650), projectedBarycentricCoords (util.cpp:313-347).
// A strictly sequential walk of a few hundred steps: one thread follows the field on the device-resident result of
// the last plan, so a makePlan moves a few KB of poses over PCIe instead of four V-sized arrays.
// ============================================================================
struct BacktrackArgs {
  const float* pos; const float* vn; const uint32_t* faces; const uint32_t* cor_ptr; const int4* cor_idx;
  const uint32_t* pred; const float* direction; const int32_t* cut;
  float start[3]; uint32_t start_face; float goal[3]; uint32_t goal_face;
  double step_width; uint32_t max_points;
  float* path_pos; uint32_t* path_face; int32_t* result /* [0] outcome, [1] n_points */; const int* cancel_flag;
  RepulsiveField layer;        // InflationLayer::vectorAt added in meshAhead (mesh_map.cpp:1097-1102); dist == null: none
  uint32_t* spill_list; uint32_t* spill_key;   // F entries each, keys all zero (bt_search_spill); null: not reserved yet
};

__device__ __forceinline__ bool projected_barycentric(F3 p, F3 a, F3 b, F3 c, float bary[3], float& dist) {
  const F3 u = f3sub(b, a), v = f3sub(c, a), w = f3sub(p, a), n = f3cross(u, v);
  const float oneOver4ASquared = (float)(1.0 / (double)f3dot(n, n));
  const float gamma = f3dot(f3cross(u, w), n) * oneOver4ASquared;
  const float beta = f3dot(f3cross(w, v), n) * oneOver4ASquared;
  const float alpha = 1 - gamma - beta;
  bary[0] = alpha; bary[1] = beta; bary[2] = gamma;
  dist = f3dot(n, w) / sqrtf(f3dot(n, n));
  const float EPSILON = 0.01f;
  return (0 - EPSILON <= alpha) && (alpha <= 1 + EPSILON) && (0 - EPSILON <= beta) && (beta <= 1 + EPSILON) &&
         (0 - EPSILON <= gamma) && (gamma <= 1 + EPSILON);
}

// One warp walks the path.  The scalar parts (position, current face, direction blend) are computed redundantly by
// all lanes; searchNeighbourFaces -- a breadth-first list of up to a few hundred faces per step -- is spread over
// the lanes 32 faces at a time: containment tests in parallel, expansions gathered per lane, deduplicated through a
// shared-memory hash set and appended in exactly the order the sequential loop of mesh_map.cpp:1031-1063 would
// produce (lane-major sequence numbers + atomicMin decide which duplicate came first), so the face that is returned
// is the same one.  A search that outgrows the shared-memory list (fine meshes: ~5000 faces per 0.4 m step at 1 cm)
// or a candidate row (a listed face next to a vertex of high degree) runs again from its start in bt_search_spill,
// which has no limit below F faces; a walk that needs it before the host reserved its workspace ends with
// BT_NEEDS_SPILL, and the host reserves it and walks again.
constexpr int32_t BT_NEEDS_SPILL = -100;   // internal outcome, never returned by the C ABI
constexpr uint32_t BT_MEMBER = 0xffffffffu;

// searchNeighbourFaces in global memory: the list in spill_list; spill_key[f] is 0 for a face not seen, BT_MEMBER for
// a listed one and, while one round of 32 listed faces is expanded, the largest key (= the first in the sequential
// order) of the candidates that name it.  Every face a round touches is listed when the round ends, so clearing the
// keys of the listed faces leaves the array all zero for the next search.  Keys are read with __ldcg: the atomics
// write them in L2.
__device__ bool bt_search_spill(const BacktrackArgs& a, F3 pos, F3 center, float rsq, uint32_t& face, float bary[3]) {
  constexpr unsigned FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x;
  uint32_t* const list = a.spill_list; uint32_t* const key = a.spill_key;
  if (lane == 0) { list[0] = face; key[face] = BT_MEMBER; }
  __syncwarp();
  uint32_t cnt = 1, it = 0;
  bool ok = false;
  while (it < cnt) {
    const uint32_t chunk = min(32u, cnt - it);
    const bool act = lane < chunk;
    const uint32_t f = act ? __ldcg(list + it + lane) : 0u;
    const uint32_t* q = a.faces + 3 * (size_t)f;
    const uint32_t qv[3] = {q[0], q[1], q[2]};
    const F3 PV[3] = {f3load(a.pos, qv[0]), f3load(a.pos, qv[1]), f3load(a.pos, qv[2])};
    float lb[3], ld;
    const bool pass = act && projected_barycentric(pos, PV[0], PV[1], PV[2], lb, ld) && fabsf(ld) < 0.4f;
    const unsigned pm = __ballot_sync(FULL, pass);
    if (pm) {
      const int L = __ffs(pm) - 1;
      face = __shfl_sync(FULL, f, L);
      bary[0] = __shfl_sync(FULL, lb[0], L); bary[1] = __shfl_sync(FULL, lb[1], L); bary[2] = __shfl_sync(FULL, lb[2], L);
      ok = true;
      break;
    }
    // my candidates: the corner rows of my vertices within the radius, in the reference's order
    uint32_t lo[3], hi[3], nc = 0;
    for (int k = 0; k < 3; ++k) {
      lo[k] = hi[k] = 0;
      const F3 e = f3sub(center, PV[k]);
      if (act && f3dot(e, e) < rsq) { lo[k] = a.cor_ptr[qv[k]]; hi[k] = a.cor_ptr[qv[k] + 1]; }
      nc += hi[k] - lo[k];
    }
    uint32_t base = nc;                                  // lane-major sequence number of my first candidate
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, base, o); if ((int)lane >= o) base += v; }
    base -= nc;
    auto key_of = [](uint32_t seq) { return BT_MEMBER - 1u - seq; };   // earlier in the sequential order: larger
    uint32_t s = base;
    for (int k = 0; k < 3; ++k)
      for (uint32_t j = lo[k]; j < hi[k]; ++j) atomicMax(&key[(uint32_t)a.cor_idx[j].z], key_of(s++));
    __syncwarp();
    uint32_t newc = 0;                                   // candidates whose key survived: the first of their face
    s = base;
    for (int k = 0; k < 3; ++k)
      for (uint32_t j = lo[k]; j < hi[k]; ++j) newc += __ldcg(&key[(uint32_t)a.cor_idx[j].z]) == key_of(s++) ? 1u : 0u;
    uint32_t incl = newc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if ((int)lane >= o) incl += v; }
    const uint32_t total = __shfl_sync(FULL, incl, 31);
    uint32_t w = cnt + incl - newc;
    s = base;                                            // append them in order; listed faces are members from now on
    for (int k = 0; k < 3; ++k)
      for (uint32_t j = lo[k]; j < hi[k]; ++j) {
        const uint32_t c = (uint32_t)a.cor_idx[j].z;
        if (__ldcg(&key[c]) == key_of(s++)) { list[w++] = c; key[c] = BT_MEMBER; }
      }
    __syncwarp();
    cnt += total; it += chunk;
  }
  for (uint32_t j = lane; j < cnt; j += 32) key[__ldcg(list + j)] = 0u;
  __syncwarp();
  return ok;
}

constexpr int BT_LIST_CAP = 4096;      // faces in the search list
constexpr int BT_HASH_CAP = 8192;      // open-addressing set over face ids (power of two)
constexpr int BT_MAXC = 64;            // expansion candidates of one listed face (<= sum of its vertices' face counts)
struct BtShared {
  uint32_t list[BT_LIST_CAP];
  uint32_t hkey[BT_HASH_CAP];
  uint32_t hseq[BT_HASH_CAP];
  uint32_t cand[32][BT_MAXC];
  uint16_t cslot[32][BT_MAXC];
};

__global__ void __launch_bounds__(32) k_backtrack(BacktrackArgs a) {
  MNB_DYNAMIC_SMEM(bt_raw);
  BtShared& S = *reinterpret_cast<BtShared*>(bt_raw);
  constexpr unsigned FULL = 0xffffffffu;
  const uint32_t lane = threadIdx.x;
  uint32_t n = 0;
  auto push = [&](F3 p, uint32_t f) {
    if (lane == 0 && n < a.max_points) { a.path_pos[3 * n] = p.x; a.path_pos[3 * n + 1] = p.y; a.path_pos[3 * n + 2] = p.z; a.path_face[n] = f; }
    ++n;
  };
  uint32_t face = a.goal_face;
  F3 pos{a.goal[0], a.goal[1], a.goal[2]};
  const F3 st{a.start[0], a.start[1], a.start[2]};
  const float step = (float)a.step_width;
  push(pos, face);
  int32_t outcome = MNB_SUCCESS;
  for (;;) {
    const F3 d = f3sub(pos, st);
    if (!((double)f3dot(d, d) > a.step_width)) break;                            // cvp:925 (distance2 vs step_width, as written)
    if (a.cancel_flag && *(volatile const int*)a.cancel_flag) { outcome = MNB_CANCELED; break; }
    if (n + 1 >= a.max_points) { outcome = MNB_E_STATE; break; }
    // ---- meshAhead ----
    float bary[3], dist;
    const uint32_t* t = a.faces + 3 * (size_t)face;
    bool ok = projected_barycentric(pos, f3load(a.pos, t[0]), f3load(a.pos, t[1]), f3load(a.pos, t[2]), bary, dist);
    if (!ok) {                                                                    // searchNeighbourFaces(pos, face, step, 0.4)
      F3 center{0, 0, 0};
      for (int k = 0; k < 3; ++k) { const F3 q = f3load(a.pos, t[k]); center = {center.x + q.x, center.y + q.y, center.z + q.z}; }
      center = {center.x / 3, center.y / 3, center.z / 3};
      float vcm = 0;
      for (int k = 0; k < 3; ++k) { const F3 e = f3sub(f3load(a.pos, t[k]), center); vcm = fmaxf(vcm, sqrtf(f3dot(e, e))); }
      const float ext = step + vcm, rsq = ext * ext;
      for (uint32_t i = lane; i < (uint32_t)BT_HASH_CAP; i += 32) { S.hkey[i] = 0xffffffffu; S.hseq[i] = 0xffffffffu; }
      __syncwarp();
      auto slot_of = [](uint32_t key) { return (key * 2654435761u) >> (32 - 13); };
      static_assert(BT_HASH_CAP == (1 << 13), "hash shift");
      if (lane == 0) {
        S.list[0] = face;
        const uint32_t h = slot_of(face); S.hkey[h] = face; S.hseq[h] = 0u;
      }
      __syncwarp();
      uint32_t cnt = 1, it = 0;
      bool overflow = false;
      while (it < cnt && !ok) {
        const uint32_t chunk = min(32u, cnt - it);
        const bool act = lane < chunk;
        const uint32_t f = act ? S.list[it + lane] : 0u;
        const uint32_t* q = a.faces + 3 * (size_t)f;
        const uint32_t q0 = q[0], q1 = q[1], q2 = q[2];
        const F3 P0 = f3load(a.pos, q0), P1 = f3load(a.pos, q1), P2 = f3load(a.pos, q2);
        float lb[3], ld;
        const bool pass = act && projected_barycentric(pos, P0, P1, P2, lb, ld) && fabsf(ld) < 0.4f;
        const unsigned pm = __ballot_sync(FULL, pass);
        if (pm) {
          const int L = __ffs(pm) - 1;
          face = __shfl_sync(FULL, f, L);
          bary[0] = __shfl_sync(FULL, lb[0], L); bary[1] = __shfl_sync(FULL, lb[1], L); bary[2] = __shfl_sync(FULL, lb[2], L);
          ok = true;
          break;
        }
        // expansion candidates of my face, in the reference's order: vertex 0, 1, 2; faces of the vertex in CSR order
        uint32_t nc = 0;
        if (act) {
          const uint32_t qv[3] = {q0, q1, q2};
          const F3 PV[3] = {P0, P1, P2};
          for (int k = 0; k < 3; ++k) {
            const F3 e = f3sub(center, PV[k]);
            if (!(f3dot(e, e) < rsq)) continue;
            for (uint32_t jx = a.cor_ptr[qv[k]]; jx < a.cor_ptr[qv[k] + 1]; ++jx) {
              if (nc < (uint32_t)BT_MAXC) S.cand[lane][nc] = (uint32_t)a.cor_idx[jx].z;
              ++nc;
            }
          }
        }
        if (__any_sync(FULL, nc > (uint32_t)BT_MAXC)) { overflow = true; break; }
        __syncwarp();
        // insert all candidates; among duplicates the smallest sequence number (= first in sequential order) wins
        for (uint32_t i = 0; i < nc; ++i) {
          const uint32_t key = S.cand[lane][i], seq = lane * (uint32_t)BT_MAXC + i + 1u;
          uint32_t h = slot_of(key);
          for (;;) {
            const uint32_t old = atomicCAS(&S.hkey[h], 0xffffffffu, key);
            if (old == 0xffffffffu || old == key) break;
            h = (h + 1u) & (uint32_t)(BT_HASH_CAP - 1);
          }
          atomicMin(&S.hseq[h], seq);
          S.cslot[lane][i] = (uint16_t)h;
        }
        __syncwarp();
        uint32_t newc = 0;
        for (uint32_t i = 0; i < nc; ++i) newc += (S.hseq[S.cslot[lane][i]] == lane * (uint32_t)BT_MAXC + i + 1u) ? 1u : 0u;
        uint32_t incl = newc;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if ((int)lane >= o) incl += v; }
        const uint32_t total = __shfl_sync(FULL, incl, 31);
        if (cnt + total > (uint32_t)BT_LIST_CAP) { overflow = true; break; }
        uint32_t w = cnt + incl - newc;
        __syncwarp();
        for (uint32_t i = 0; i < nc; ++i) {
          const uint32_t h = S.cslot[lane][i];
          if (S.hseq[h] == lane * (uint32_t)BT_MAXC + i + 1u) S.list[w++] = S.cand[lane][i];
        }
        __syncwarp();
        for (uint32_t i = 0; i < nc; ++i) {            // commit: members of the list can never be "new" again
          const uint32_t h = S.cslot[lane][i];
          if (S.hseq[h] == lane * (uint32_t)BT_MAXC + i + 1u) S.hseq[h] = 0u;
        }
        __syncwarp();
        cnt += total; it += chunk;
      }
      if (overflow) {
        if (!a.spill_list) { outcome = BT_NEEDS_SPILL; break; }
        ok = bt_search_spill(a, pos, center, rsq, face, bary);
      }
      if (!ok) { outcome = MNB_NO_PATH_FOUND; break; }
      t = a.faces + 3 * (size_t)face;
      const F3 A = f3load(a.pos, t[0]), B = f3load(a.pos, t[1]), C = f3load(a.pos, t[2]);   // project onto the surface
      pos = {A.x * bary[0] + B.x * bary[1] + C.x * bary[2], A.y * bary[0] + B.y * bary[1] + C.y * bary[2],
             A.z * bary[0] + B.z * bary[1] + C.z * bary[2]};
    }
    // ---- directionAtPosition ----
    bool any = false;
    F3 vec{0, 0, 0};
    for (int k = 0; k < 3; ++k) {
      F3 e;
      if (!vertex_vector(a.pos, a.vn, a.pred, a.direction, a.cut, t[k], e)) continue;
      any = true;
      vec = {vec.x + e.x * bary[k], vec.y + e.y * bary[k], vec.z + e.z * bary[k]};
    }
    if (!any || !(isfinite(vec.x) && isfinite(vec.y) && isfinite(vec.z))) { outcome = MNB_NO_PATH_FOUND; break; }
    F3 dir = f3normalized(vec);                          // opt_dir.get().normalized()
    if (a.layer.dist) { const F3 lv = inflation_vector_at(a.layer, t, bary); dir = F3{dir.x + lv.x, dir.y + lv.y, dir.z + lv.z}; }
    dir = f3normalized(dir);                             // dir += layer->vectorAt(...); dir.normalize()
    pos = {pos.x + dir.x * step, pos.y + dir.y * step, pos.z + dir.z * step};
    push(pos, face);
  }
  if (outcome == MNB_SUCCESS) push(st, a.start_face);                            // cvp:951
  if (lane == 0) { a.result[0] = outcome; a.result[1] = (int32_t)n; }
}

// ============================================================================
// Localisation: MeshMap::getNearestVertexHandle (mesh_map.cpp:1161-1174; the reference walks a nanoflann KD-tree,
// here the 12 B/vertex position array is streamed once for ALL queries of the call -- HBM-bound, ~8 us per 5M-vertex
// pass) and MeshMap::searchContainingFace (mesh_map.cpp:1120-1159).
// Key = (squared distance bits << 32) | vertex id: non-negative floats order like their bit patterns, so one 64-bit
// atomicMin yields the nearest vertex with ties to the lowest id.
// ============================================================================
constexpr int LOC_Q = 32;       // queries per pass (registers)

__global__ void __launch_bounds__(256) k_nearest_vertex(const float* __restrict__ pos, uint32_t V, const float* __restrict__ points,
                                                        uint32_t q0, uint32_t nq, unsigned long long* __restrict__ keys) {
  __shared__ float sq[3 * LOC_Q];
  __shared__ unsigned long long sbest[LOC_Q];
  if (threadIdx.x < 3 * nq) sq[threadIdx.x] = points[3 * (size_t)q0 + threadIdx.x];
  if (threadIdx.x < LOC_Q) sbest[threadIdx.x] = ~0ull;
  __syncthreads();
  unsigned long long best[LOC_Q];
#pragma unroll
  for (int q = 0; q < LOC_Q; ++q) best[q] = ~0ull;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) {
    const float x = pos[3 * (size_t)v], y = pos[3 * (size_t)v + 1], z = pos[3 * (size_t)v + 2];
#pragma unroll
    for (int q = 0; q < LOC_Q; ++q) {
      if (q < (int)nq) {
        const float dx = sq[3 * q] - x, dy = sq[3 * q + 1] - y, dz = sq[3 * q + 2] - z;
        const float d = dx * dx + dy * dy + dz * dz;
        const unsigned long long key = ((unsigned long long)__float_as_uint(d) << 32) | v;
        if (!(d != d) && key < best[q]) best[q] = key;
      }
    }
  }
#pragma unroll
  for (int q = 0; q < LOC_Q; ++q) {
    if (q < (int)nq) {
      unsigned long long b = best[q];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, b, o); b = t < b ? t : b; }
      if ((threadIdx.x & 31) == 0 && b != ~0ull) atomicMin(&sbest[q], b);
    }
  }
  __syncthreads();
  if (threadIdx.x < nq && sbest[threadIdx.x] != ~0ull) atomicMin(&keys[q0 + threadIdx.x], sbest[threadIdx.x]);
}

__global__ void k_containing_face(const float* __restrict__ pos, const uint32_t* __restrict__ faces, const uint32_t* __restrict__ cor_ptr,
                                  const int4* __restrict__ cor_idx, const float* __restrict__ points, uint32_t n,
                                  const unsigned long long* __restrict__ keys, uint32_t* __restrict__ out_vertex,
                                  int32_t* __restrict__ out_face, float* __restrict__ out_bary) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const uint32_t best = (uint32_t)(keys[q] & 0xffffffffu);
  if (out_vertex) out_vertex[q] = best;
  const F3 p = f3load(points, q);
  float lowest = 3.402823466e+38f;
  int32_t bf = -1; float bb[3] = {0, 0, 0};
  for (uint32_t k = cor_ptr[best]; k < cor_ptr[best + 1]; ++k) {
    const uint32_t f = (uint32_t)cor_idx[k].z;
    const uint32_t* t = faces + 3 * (size_t)f;
    float cb[3], dist = 0;
    if (projected_barycentric(p, f3load(pos, t[0]), f3load(pos, t[1]), f3load(pos, t[2]), cb, dist) && dist < lowest) {
      lowest = dist; bf = (int32_t)f; bb[0] = cb[0]; bb[1] = cb[1]; bb[2] = cb[2];
    }
  }
  if (out_face) out_face[q] = bf;
  if (out_bary) { out_bary[3 * (size_t)q] = bb[0]; out_bary[3 * (size_t)q + 1] = bb[1]; out_bary[3 * (size_t)q + 2] = bb[2]; }
}
