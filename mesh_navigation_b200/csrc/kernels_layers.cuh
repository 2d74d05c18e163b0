// Fused geometric cost layers + MaxCombination + lethal masks, face / vertex normals.
// (part of libmeshnav_b200.so: included by meshnav.cu, which holds the C ABI and all host code)
#pragma once
#include "launch.cuh"
#include "../../include/meshnav_b200.h"
#include "band_engine.cuh"
#include <type_traits>

using namespace mnb;

// ============================================================================
// Fused geometric cost layers (mesh_layers: HeightDiff, Roughness, Steepness, Ridge, Clearance cost
// mapping, Border) + MaxCombinationLayer + lethal masks: ONE pass over the radius neighbourhood per
// vertex instead of the reference's three independent visitLocalVertexNeighborhood runs with
// std::set bookkeeping (ridge_layer.cpp:166-175, height_diff_layer.cpp:108, roughness_layer.cpp:143).
// Definitions of the lvr2 pieces: see oracle/oracle.cpp (orc_layers).
// ============================================================================
__global__ void k_face_normals(const float* __restrict__ pos, const uint32_t* __restrict__ faces, uint32_t F,
                               float* __restrict__ fn) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const float* p0 = pos + 3 * (size_t)faces[3 * (size_t)f];
  const float* p1 = pos + 3 * (size_t)faces[3 * (size_t)f + 1];
  const float* p2 = pos + 3 * (size_t)faces[3 * (size_t)f + 2];
  const float ax = p1[0] - p0[0], ay = p1[1] - p0[1], az = p1[2] - p0[2];
  const float bx = p2[0] - p0[0], by = p2[1] - p0[1], bz = p2[2] - p0[2];
  float nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
  const float l = sqrtf(nx * nx + ny * ny + nz * nz);
  if (l > 0) { nx /= l; ny /= l; nz /= l; }
  fn[3 * (size_t)f] = nx; fn[3 * (size_t)f + 1] = ny; fn[3 * (size_t)f + 2] = nz;
}

__global__ void k_vertex_normals(const uint32_t* __restrict__ cor_ptr, const int4* __restrict__ cor_idx,
                                 const float* __restrict__ fn, uint32_t V, float* __restrict__ vn) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  float nx = 0, ny = 0, nz = 0;
  for (uint32_t k = cor_ptr[v]; k < cor_ptr[v + 1]; ++k) {
    const int f = cor_idx[k].z;
    nx = nx + fn[3 * (size_t)f]; ny = ny + fn[3 * (size_t)f + 1]; nz = nz + fn[3 * (size_t)f + 2];
  }
  const float l = sqrtf(nx * nx + ny * ny + nz * nz);
  if (l > 0) { nx /= l; ny /= l; nz /= l; }
  vn[3 * (size_t)v] = nx; vn[3 * (size_t)v + 1] = ny; vn[3 * (size_t)v + 2] = nz;
}

// acos of a float as the layers use it (roughness: angle between normals, steepness_layer.cpp:165): evaluated in double and
// rounded once.  The reference calls the float overload of its libm, whose last bit differs between libm versions and
// from CUDA's acosf; lethal sets are threshold tests on these values, so both this kernel and the oracle use the value
// that is well defined everywhere -- the correctly rounded one (double acos is accurate to < 2 ulp of double on both sides).
__device__ __forceinline__ float acos_f(float x) { return (float)acos((double)x); }

struct LayerKernelArgs {
  uint32_t V;
  const float* pos; const float* vn;
  const uint32_t* adj_ptr; const uint32_t* adj_nbr;
  const uint8_t* border;
  const float* clearance;      // may be null
  mnb_layer_params P;
  float* costs;                // 6 x V
  float* combined; uint8_t* lethal_mask;
  unsigned int* overflow;      // neighbourhood larger than the per-thread scratch
  // packed copies for the prefetching walk: one 16-byte load per position / normal, one 32-byte row of neighbour ids per vertex
  const float4* pos4; const float4* vn4; const uint4* nbr8;
};

// The prefetching walk reads packed copies of the same data: every per-thread (scattered) load instruction costs 32 L1
// wavefronts whatever its width, so {x,y,z} as three 4-byte loads and a neighbour list behind two CSR pointers triple the
// wavefront count of the walk, which is what bounds the kernel (DESIGN.md 5).
constexpr uint32_t NBR8_EMPTY = 0xffffffffu, NBR8_BIG = 0xfffffffeu;
__global__ void k_pack_layers(const float* __restrict__ pos, const float* __restrict__ vn, const uint32_t* __restrict__ adj_ptr,
                              const uint32_t* __restrict__ adj_nbr, uint32_t V, float4* __restrict__ pos4, float4* __restrict__ vn4,
                              uint32_t* __restrict__ nbr8) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  pos4[v] = make_float4(pos[3 * (size_t)v], pos[3 * (size_t)v + 1], pos[3 * (size_t)v + 2], 0.0f);
  vn4[v] = make_float4(vn[3 * (size_t)v], vn[3 * (size_t)v + 1], vn[3 * (size_t)v + 2], 0.0f);
  const uint32_t kb = adj_ptr[v], deg = adj_ptr[v + 1] - kb;
  for (uint32_t j = 0; j < 8; ++j)      // CSR order (ascending edge id) is kept: the traversal order must not change
    nbr8[8 * (size_t)v + j] = deg > 8 ? NBR8_BIG : (j < deg ? adj_nbr[kb + j] : NBR8_EMPTY);
}

__device__ __forceinline__ float3 load3(const float* p, uint32_t v) { return make_float3(p[3 * (size_t)v], p[3 * (size_t)v + 1], p[3 * (size_t)v + 2]); }
__device__ __forceinline__ float3 xyz(const float4& q) { return make_float3(q.x, q.y, q.z); }

// The accumulators of the three radius layers, carried through the walks of one vertex (with the counts first, ptxas
// gives the prefetching kernels the registers and stack of the separate variables this replaced, and no spills)
struct LayerSums { int rcnt, num; float zmin, zmax, rsum, value; };

// What every form of the neighbourhood walk shares: the centre vertex, the radius, and the step for a newly seen neighbour.
// WHICH selects the accumulators that are active (bit0 height diff, bit1 roughness, bit2 ridge) so that layers with equal
// radii share one walk.  The forms differ only in where a neighbour's position and normal come from and in how the seen-set
// and the stack are stored; the float operations and their order are these, so all forms give bit-identical sums.
template <int WHICH>
struct WalkCentre {
  float radius, px, py, pz, nvx, nvy, nvz, rx, ry, rz;
  __device__ __forceinline__ WalkCentre(float radius, float3 p, float3 n)
      : radius(radius), px(p.x), py(p.y), pz(p.z), nvx(n.x), nvy(n.y), nvz(n.z), rx(p.x + n.x), ry(p.y + n.y), rz(p.z + n.z) {}
  // neighbour at q, its normal from normal() (called only when an active layer needs it): adds it to s and returns true
  // when it lies inside the radius, i.e. when the walk continues through it
  template <class Normal>
  __device__ __forceinline__ bool add(LayerSums& s, float3 q, Normal normal) const {
    const float dx = q.x - px, dy = q.y - py, dz = q.z - pz;
    if (!(sqrtf(dx * dx + dy * dy + dz * dz) < radius)) return false;
    if (WHICH & 1) { s.zmin = fminf(s.zmin, q.z); s.zmax = fmaxf(s.zmax, q.z); }
    if (WHICH & 6) {
      const float3 nn = normal();
      if (WHICH & 2) {
        float dot = nvx * nn.x + nvy * nn.y + nvz * nn.z;
        dot = fminf(1.0f, fmaxf(-1.0f, dot));
        s.rsum = s.rsum + acos_f(dot); s.rcnt++;
      }
      if (WHICH & 4) {
        const float cx = (q.x + nn.x) - rx, cy = (q.y + nn.y) - ry, cz = (q.z + nn.z) - rz;
        s.value += sqrtf(cx * cx + cy * cy + cz * cz); s.num++;
      }
    }
    return true;
  }
};

constexpr int NB_SEEN = 320, NB_STACK = 160;

// (fallback for neighbourhoods that overflow the hashed sets below: linear `seen` list, any size up to NB_SEEN)
template <int WHICH>
__device__ __noinline__ void walk_linear(const LayerKernelArgs& a, uint32_t v, float radius, LayerSums& s) {
  uint32_t seen[NB_SEEN]; uint32_t stack[NB_STACK];
  int ns = 0, sp = 0;
  seen[ns++] = v; stack[sp++] = v;
  const WalkCentre<WHICH> c(radius, load3(a.pos, v), load3(a.vn, v));
  while (sp > 0) {
    const uint32_t u = stack[--sp];
    for (uint32_t k = a.adj_ptr[u]; k < a.adj_ptr[u + 1]; ++k) {
      const uint32_t n = a.adj_nbr[k];
      bool was = false;
      for (int i = 0; i < ns; ++i) if (seen[i] == n) { was = true; break; }
      if (was) continue;
      if (ns >= NB_SEEN) { atomicAdd(a.overflow, 1u); return; }
      seen[ns++] = n;
      if (c.add(s, load3(a.pos, n), [&] { return load3(a.vn, n); })) {
        if (sp >= NB_STACK) { atomicAdd(a.overflow, 1u); return; }
        stack[sp++] = n;
      }
    }
  }
}

// Same traversal, same visiting order (so the float sums are bit-identical to the oracle's), but the `seen` set is a
// 128-entry open-addressing hash in local memory instead of a linear list: ~2 probes per membership test instead of
// ~24 compares.  Neighbourhoods with more than NB_HSEEN seen vertices fall back to walk_linear.
constexpr int NB_HASH = 128, NB_HSEEN = 96;
__device__ __forceinline__ uint32_t seen_slot(uint32_t n) { return (n * 2654435761u) >> 25; }
template <int WHICH>
__device__ __forceinline__ void walk(const LayerKernelArgs& a, uint32_t v, float radius, LayerSums& s) {
  uint32_t ht[NB_HASH]; uint32_t stack[NB_HSEEN];
#pragma unroll 8
  for (int i = 0; i < NB_HASH; ++i) ht[i] = 0xffffffffu;
  const LayerSums s0 = s;
  int ns = 0, sp = 0;
  ht[seen_slot(v)] = v; ns = 1; stack[sp++] = v;
  const WalkCentre<WHICH> c(radius, load3(a.pos, v), load3(a.vn, v));
  bool overflow = false;
  while (sp > 0 && !overflow) {
    const uint32_t u = stack[--sp];
    for (uint32_t k = a.adj_ptr[u]; k < a.adj_ptr[u + 1]; ++k) {
      const uint32_t n = a.adj_nbr[k];
      uint32_t h = seen_slot(n);
      bool was = false;
      for (;;) {
        const uint32_t e = ht[h];
        if (e == n) { was = true; break; }
        if (e == 0xffffffffu) break;
        h = (h + 1u) & (uint32_t)(NB_HASH - 1);
      }
      if (was) continue;
      if (ns >= NB_HSEEN) { overflow = true; break; }
      ht[h] = n; ++ns;
      if (c.add(s, load3(a.pos, n), [&] { return load3(a.vn, n); }))
        stack[sp++] = n;            // sp <= ns <= NB_HSEEN
    }
  }
  if (overflow) { s = s0; walk_linear<WHICH>(a, v, radius, s); }
}

// The prefetching walk runs PF_THREADS threads per CTA; each keeps its seen-set and a stack of PF_STACK entries in shared
// memory, slot-major (entry i of thread t at [i * PF_THREADS + t]: conflict free).  Two forms of the seen-set:
//  * Key = uint32_t: the hash holds vertex ids, the stack vertex ids (704 bytes per thread);
//  * Key = uint16_t, the compact form: the hash holds 16-bit codes  n - v + 32768  relative to the centre v (0 = empty), the
//    stack the 8-bit hash slot of a vertex (304 bytes per thread).  The 704 bytes of the 32-bit form cap the kernel at 10
//    resident warps per SM, and it is bound by instruction issue at that occupancy (ncu: 34 % issue utilisation at 15 %
//    active warps); the compact form allows 18.  Vertex ids inside one neighbourhood are close to the centre's on any mesh
//    whose numbering has spatial locality (scan order, Morton order, most reconstruction outputs); a neighbour whose id is
//    further than 32767 from the centre's counts as an overflow of the set, so that vertex is redone by walk_linear.
constexpr int PF_THREADS = 64, PF_STACK = 48;
template <class K>
struct SharedSeen {
  using Key = K;
  static constexpr bool COMPACT = sizeof(Key) == 2;
  using Entry = std::conditional_t<COMPACT, uint8_t, uint32_t>;
  static constexpr Key EMPTY = COMPACT ? 0 : 0xffffffffu;
  static constexpr size_t BYTES = NB_HASH * sizeof(Key) + PF_STACK * sizeof(Entry);     // per thread
  Key* ht; Entry* stack; uint32_t v;
  __device__ __forceinline__ SharedSeen(unsigned char* smem, uint32_t v)
      : ht(reinterpret_cast<Key*>(smem) + threadIdx.x),
        stack(reinterpret_cast<Entry*>(smem + NB_HASH * sizeof(Key) * PF_THREADS) + threadIdx.x), v(v) {}
  __device__ __forceinline__ Key& slot(uint32_t h) const { return ht[h * PF_THREADS]; }
  // a new walk: the set holds the centre v alone, the stack v
  __device__ __forceinline__ void start() const {
#pragma unroll 8
    for (int i = 0; i < NB_HASH; ++i) slot(i) = EMPTY;
    const uint32_t h0 = seen_slot(v);
    Key k; key(v, k); slot(h0) = k; push(0, v, h0);
  }
  // the key of vertex n; false when n is out of the compact form's range
  __device__ __forceinline__ bool key(uint32_t n, Key& k) const {
    if constexpr (!COMPACT) { k = n; return true; }
    const uint32_t code = n - v + 32768u;                     // wraps for n < v; in range <=> 1 <= code <= 65535
    k = (Key)code;
    return code - 1u < 65535u;
  }
  // stack entry i: vertex n, which the hash holds in slot h
  __device__ __forceinline__ void push(int i, uint32_t n, uint32_t h) const { stack[i * PF_THREADS] = (Entry)(COMPACT ? h : n); }
  __device__ __forceinline__ uint32_t pop(int i) const {
    if constexpr (!COMPACT) return stack[i * PF_THREADS];
    return v + (uint32_t)slot((uint32_t)stack[i * PF_THREADS]) - 32768u;
  }
};

// The same traversal (same visiting order, same sums) with memory-level parallelism instead of occupancy.  The walk is a
// chain of dependent loads -- pop u, load u's neighbour row, then per neighbour: hash probe -> position -> (inside the
// radius) normal -- ~13 L2 round trips per expanded vertex, which is what the 9.6 ms of the per-thread form were made of
// (round 2 ncu: 18 % issue utilisation, everything on the long scoreboard; a shared-memory hash alone changed nothing).
// Here the positions AND normals of all (up to 8) neighbours of u are requested up front, 16 independent 16-byte loads in
// flight per thread, before the first hash probe; the sequential part then runs on registers.
template <int WHICH, class Seen>
__device__ __forceinline__ void walk_pf(const LayerKernelArgs& a, uint32_t v, float radius, LayerSums& s, const Seen& seen) {
  seen.start();
  const LayerSums s0 = s;
  int ns = 1, sp = 1;
  const WalkCentre<WHICH> c(radius, xyz(__ldg(&a.pos4[v])), xyz(__ldg(&a.vn4[v])));
  bool overflow = false;
  auto visit = [&](uint32_t n, const float4& q, const float4& nn) {
    typename Seen::Key k;
    if (!seen.key(n, k)) { overflow = true; return; }
    uint32_t h = seen_slot(n);
    for (;;) {
      const auto e = seen.slot(h);
      if (e == k) return;
      if (e == Seen::EMPTY) break;
      h = (h + 1u) & (uint32_t)(NB_HASH - 1);
    }
    if (ns >= NB_HSEEN) { overflow = true; return; }
    seen.slot(h) = k; ++ns;
    if (!c.add(s, xyz(q), [&] { return xyz(nn); })) return;
    if (sp >= PF_STACK) { overflow = true; return; }
    seen.push(sp++, n, h);
    mnb_prefetch_l2(a.nbr8 + 2 * (size_t)n);   // its row is needed when it is popped
  };
  while (sp > 0 && !overflow) {
    const uint32_t u = seen.pop(--sp);
    const uint4 r0 = __ldg(&a.nbr8[2 * (size_t)u]);
    if (r0.x == NBR8_BIG) {                       // more than 8 neighbours: CSR row, one at a time
      for (uint32_t k = a.adj_ptr[u]; k < a.adj_ptr[u + 1] && !overflow; ++k) { const uint32_t n = a.adj_nbr[k]; visit(n, __ldg(&a.pos4[n]), __ldg(&a.vn4[n])); }
      continue;
    }
    const uint4 r1 = __ldg(&a.nbr8[2 * (size_t)u + 1]);
    const uint32_t ids[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
    float4 q[8], nn[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {                 // all requests first ...
      const uint32_t n = ids[j] == NBR8_EMPTY ? v : ids[j];
      q[j] = __ldg(&a.pos4[n]);
      if (WHICH & 6) nn[j] = __ldg(&a.vn4[n]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {                 // ... then the sequential part, in the reference's order
      if (ids[j] == NBR8_EMPTY || overflow) break;
      visit(ids[j], q[j], nn[j]);
    }
  }
  if (overflow) { s = s0; walk_linear<WHICH>(a, v, radius, s); }
}

// per-vertex layer values from the accumulators of the walks, lethal bits, MaxCombination
__device__ __forceinline__ void layers_epilogue(const LayerKernelArgs& a, uint32_t v, const LayerSums& s) {
  const mnb_layer_params& P = a.P;
  const float hd = s.zmax - s.zmin;
  const float ro = s.rcnt ? s.rsum / (float)s.rcnt : 0.0f;
  const float st = acos_f(a.vn[3 * (size_t)v + 2]);                               // steepness_layer.cpp:165
  const float ri = s.num == 0 ? (float)(P.ridge_threshold + 0.1) : s.value / s.num;     // ridge_layer.cpp:177-184
  const float cl = a.clearance ? a.clearance[v] : __uint_as_float(INF_BITS);
  float cc; bool cl_lethal = false;                                              // clearance_layer.cpp:77-96
  const double inflated_height = P.clearance_robot_height + P.clearance_height_inflation;
  if (cl < P.clearance_robot_height) { cc = 1.0f; cl_lethal = true; }
  else if (cl < inflated_height) {
    const double diff = (cl - P.clearance_robot_height) / P.clearance_height_inflation;
    cc = (float)((cos(diff * 3.14159265358979323846) + 1.0) / 2.0);
  } else cc = 0.0f;
  const float bo = a.border[v] ? (float)P.border_cost : 0.0f;
  const size_t V = a.V;
  if (a.costs) {
    a.costs[v] = hd; a.costs[V + v] = ro; a.costs[2 * V + v] = st; a.costs[3 * V + v] = ri; a.costs[4 * V + v] = cc; a.costs[5 * V + v] = bo;
  }
  uint8_t mask = 0;
  if (hd > P.height_diff_threshold) mask |= 1;
  if (ro > P.roughness_threshold) mask |= 2;
  if (st > P.steepness_threshold) mask |= 4;
  if (ri > P.ridge_threshold) mask |= 8;
  if (cl_lethal) mask |= 16;
  if (bo > P.border_threshold) mask |= 32;
  if (a.lethal_mask) a.lethal_mask[v] = mask;
  if (a.combined) a.combined[v] = fmaxf(fmaxf(fmaxf(0.0f, hd), fmaxf(ro, st)), fmaxf(fmaxf(ri, cc), bo));   // combination_layer.cpp:60-71
}

// The walks k_layers<WALK> is built for; the numbers are the modes of mnb_debug_set_layers_smem.  LOCAL: walk, thread-local
// seen-set (LOCAL_THREADS per CTA), the reference the tests compare the others with; PF32 / PF16: walk_pf with the 32-bit /
// the compact seen-set (PF_THREADS per CTA, dynamic shared memory PF_THREADS x SharedSeen<Key>::BYTES).  mnb_set_mesh picks
// PF16 when the mesh's numbering keeps neighbourhoods within its range, PF32 otherwise.
constexpr int LAYERS_WALK_LOCAL = 0, LAYERS_WALK_PF32 = 2, LAYERS_WALK_PF16 = 5;
constexpr int LOCAL_THREADS = 128;

template <int WALK, int WHICH>
__device__ __forceinline__ void layer_walk(const LayerKernelArgs& a, uint32_t v, float radius, LayerSums& s, unsigned char* smem) {
  if constexpr (WALK == LAYERS_WALK_LOCAL) walk<WHICH>(a, v, radius, s);
  else walk_pf<WHICH>(a, v, radius, s, SharedSeen<std::conditional_t<WALK == LAYERS_WALK_PF16, uint16_t, uint32_t>>(smem, v));
}

// one thread per vertex: one walk when the three radius layers have equal radii, one per layer otherwise
template <int WALK>
__global__ void __launch_bounds__(WALK == LAYERS_WALK_LOCAL ? LOCAL_THREADS : PF_THREADS) k_layers(const LayerKernelArgs a) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.V) return;
  const mnb_layer_params& P = a.P;
  const float pz = a.pos[3 * (size_t)v + 2];
  LayerSums s{0, 0, pz, pz, 0.0f, 0.0f};
  const float r_hd = (float)P.height_diff_radius, r_ro = (float)P.roughness_radius, r_ri = (float)P.ridge_radius;
  MNB_DYNAMIC_SMEM(smem);
  if (r_hd == r_ro && r_ro == r_ri) {
    layer_walk<WALK, 7>(a, v, r_hd, s, smem);
  } else {
    layer_walk<WALK, 1>(a, v, r_hd, s, smem);
    layer_walk<WALK, 2>(a, v, r_ro, s, smem);
    layer_walk<WALK, 4>(a, v, r_ri, s, smem);
  }
  layers_epilogue(a, v, s);
}
