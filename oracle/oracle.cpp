// ============================================================================
// oracle/oracle.cpp  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Dependency-free CPU restatement of the reference's wavefront hot path
// (naturerobots/mesh_navigation @ b9f2851).  Only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / --impl reference legs may load this file's
// shared object.  The product library (mesh_navigation_b200/csrc) never links,
// loads or calls it.
//
// Every function cites the reference file:line it follows.  The reference's TUs
// include <lvr2/...> and <rclcpp/...> (neither is on this machine, SURVEY.md 8c)
// so the reference cannot be compiled here; this file restates the arithmetic
// with flat arrays standing in for the lvr2 attribute maps and an indexed binary
// min-heap standing in for lvr2::Meap (un-vendored dependency lvr2 @ "main",
// source_dependencies.yaml:4-7).
//
// PARITY PINNING
//   pinned by the reference's own tests (mesh_layers/test/inflation_layer_test.cpp):
//     * InflationLayer::waveFrontUpdate on the single triangle -> true, d[v2]==0.5f
//     * InflationLayer::fading table (0.2->0.9, 0.5->0.9, 0<f(0.6)<0.9, 2.0->0)
//   everything else (Dijkstra, CVP, waveCostInflation as a whole, edge weights,
//   the geometric layers, lvr2::Meap tie order, lvr2 circulator order):
//   PARITY UNPINNED -- the reference holds no test or golden vector for them;
//   parity is defined against this restatement (DESIGN.md says the same).
//
// Canonical orders replacing lvr2 circulators (results depend on them only for
// exact float ties and the inflation vector-field accumulation):
//   faces of a vertex  : ascending face id
//   edges of a vertex  : ascending edge id
// Build: g++ -O3 -ffp-contract=off  (the reference builds for generic x86-64, no
// FMA contraction; keep expression evaluation identical).
// ============================================================================
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <unordered_set>
#include <vector>

namespace {

constexpr float FINF = std::numeric_limits<float>::infinity();

// ---------------------------------------------------------------------------
// lvr2::Meap<VertexHandle,float> restated (lvr2/util/Meap.hpp, un-vendored).
// Array binary min-heap + key->slot index.  insert() on a present key updates
// the value and re-sifts (relied on at cvp_mesh_planner.cpp:814,
// dijkstra_mesh_planner.cpp:335, inflation_layer.cpp:452).  Strict '<' sifts.
// ---------------------------------------------------------------------------
struct Meap {
  struct Item { uint32_t key; float value; };
  std::vector<Item> heap;
  std::vector<int32_t> slot;  // -1 = absent
  // canonical_ties = false: plain value comparison (lvr2::Meap as restated; pop order among
  //   bit-identical float keys then depends on heap history -- unpinned, SURVEY.md H2).
  // canonical_ties = true : ties between bit-identical keys pop in ascending vertex index.  This
  //   makes the result independent of heap internals; the GPU path implements the same rule.
  bool canonical_ties;
  explicit Meap(uint32_t n, bool canonical = false) : slot(n, -1), canonical_ties(canonical) {}
  bool less(const Item& a, const Item& b) const {
    return a.value < b.value || (canonical_ties && a.value == b.value && a.key < b.key);
  }
  bool isEmpty() const { return heap.empty(); }
  void swapSlots(size_t a, size_t b) {
    std::swap(heap[a], heap[b]);
    slot[heap[a].key] = (int32_t)a;
    slot[heap[b].key] = (int32_t)b;
  }
  void bubbleUp(size_t idx) {
    while (idx != 0) {
      size_t father = (idx - 1) / 2;
      if (less(heap[idx], heap[father])) { swapSlots(idx, father); idx = father; }
      else break;
    }
  }
  void bubbleDown(size_t idx) {
    const size_t n = heap.size();
    for (;;) {
      size_t l = 2 * idx + 1, r = 2 * idx + 2, s = idx;
      if (l < n && less(heap[l], heap[s])) s = l;
      if (r < n && less(heap[r], heap[s])) s = r;
      if (s == idx) break;
      swapSlots(idx, s);
      idx = s;
    }
  }
  void insert(uint32_t key, float value) {
    int32_t s = slot[key];
    if (s >= 0) {
      float old = heap[s].value;
      heap[s].value = value;
      if (value > old) bubbleDown((size_t)s); else bubbleUp((size_t)s);
      return;
    }
    heap.push_back({key, value});
    slot[key] = (int32_t)(heap.size() - 1);
    bubbleUp(heap.size() - 1);
  }
  Item popMin() {
    Item top = heap[0];
    swapSlots(0, heap.size() - 1);
    heap.pop_back();
    slot[top.key] = -1;
    if (!heap.empty()) bubbleDown(0);
    return top;
  }
};

struct OrcMesh {
  uint32_t V = 0, F = 0, E = 0;
  std::vector<float> pos;           // 3V
  std::vector<uint32_t> faces;      // 3F, cyclic order as given
  std::vector<uint32_t> edges;      // 2E, (lo, hi)
  std::vector<uint32_t> face_edges; // 3F: edge(v0,v1), edge(v1,v2), edge(v2,v0)
  std::vector<uint32_t> ve_ptr, ve_edge, ve_nbr;  // vertex -> incident edges
  std::vector<uint32_t> vf_ptr, vf_face;          // vertex -> incident faces
  std::vector<int32_t> edge_faces;                // 2E, -1 = none
};

inline uint64_t ekey(uint32_t a, uint32_t b) {
  uint32_t lo = a < b ? a : b, hi = a < b ? b : a;
  return ((uint64_t)lo << 32) | hi;
}

void buildTopology(OrcMesh& m, const uint32_t* edges_in, uint32_t E_in) {
  const uint32_t V = m.V, F = m.F;
  // edges
  std::vector<uint64_t> keys;
  if (edges_in) {
    keys.resize(E_in);
    for (uint32_t e = 0; e < E_in; ++e) keys[e] = ekey(edges_in[2 * e], edges_in[2 * e + 1]);
    m.E = E_in;
    m.edges.assign(edges_in, edges_in + 2 * (size_t)E_in);
  } else {
    keys.reserve(3 * (size_t)F);
    for (uint32_t f = 0; f < F; ++f) {
      const uint32_t* v = &m.faces[3 * (size_t)f];
      keys.push_back(ekey(v[0], v[1]));
      keys.push_back(ekey(v[1], v[2]));
      keys.push_back(ekey(v[2], v[0]));
    }
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    m.E = (uint32_t)keys.size();
    m.edges.resize(2 * (size_t)m.E);
    for (uint32_t e = 0; e < m.E; ++e) {
      m.edges[2 * (size_t)e] = (uint32_t)(keys[e] >> 32);
      m.edges[2 * (size_t)e + 1] = (uint32_t)(keys[e] & 0xffffffffu);
    }
  }
  // key -> edge id lookup (sorted copy with ids when caller supplied the order)
  std::vector<std::pair<uint64_t, uint32_t>> lut(m.E);
  for (uint32_t e = 0; e < m.E; ++e) lut[e] = {ekey(m.edges[2 * (size_t)e], m.edges[2 * (size_t)e + 1]), e};
  std::sort(lut.begin(), lut.end());
  auto find_edge = [&](uint32_t a, uint32_t b) -> uint32_t {
    uint64_t k = ekey(a, b);
    auto it = std::lower_bound(lut.begin(), lut.end(), std::make_pair(k, (uint32_t)0));
    return it->second;
  };
  m.face_edges.resize(3 * (size_t)F);
  m.edge_faces.assign(2 * (size_t)m.E, -1);
  {
    // edge of every half-edge: sort the 3F (key, slot) pairs once and walk them against the sorted edge keys (same result
    // as a find_edge() binary search per half-edge, several times faster on multi-million-vertex meshes)
    std::vector<std::pair<uint64_t, uint32_t>> half(3 * (size_t)F);
    for (uint32_t f = 0; f < F; ++f) {
      const uint32_t* v = &m.faces[3 * (size_t)f];
      for (int k = 0; k < 3; ++k) half[3 * (size_t)f + k] = {ekey(v[k], v[(k + 1) % 3]), 3 * f + (uint32_t)k};
    }
    std::sort(half.begin(), half.end());
    size_t c = 0;
    for (const auto& h : half) {
      while (c < lut.size() && lut[c].first < h.first) ++c;
      m.face_edges[h.second] = (c < lut.size() && lut[c].first == h.first) ? lut[c].second : find_edge(h.first >> 32, (uint32_t)h.first);
    }
  }
  for (uint32_t f = 0; f < F; ++f) {            // faces in ascending id: the lower face id takes side 0 of an edge
    for (int k = 0; k < 3; ++k) {
      const uint32_t e = m.face_edges[3 * (size_t)f + k];
      if (m.edge_faces[2 * (size_t)e] < 0) m.edge_faces[2 * (size_t)e] = (int32_t)f;
      else m.edge_faces[2 * (size_t)e + 1] = (int32_t)f;
    }
  }
  // vertex -> edges (ascending edge id)
  m.ve_ptr.assign((size_t)V + 1, 0);
  for (uint32_t e = 0; e < m.E; ++e) { m.ve_ptr[m.edges[2 * (size_t)e] + 1]++; m.ve_ptr[m.edges[2 * (size_t)e + 1] + 1]++; }
  for (uint32_t v = 0; v < V; ++v) m.ve_ptr[v + 1] += m.ve_ptr[v];
  m.ve_edge.resize(m.ve_ptr[V]); m.ve_nbr.resize(m.ve_ptr[V]);
  {
    std::vector<uint32_t> cur(m.ve_ptr.begin(), m.ve_ptr.end() - 1);
    for (uint32_t e = 0; e < m.E; ++e) {
      uint32_t a = m.edges[2 * (size_t)e], b = m.edges[2 * (size_t)e + 1];
      m.ve_edge[cur[a]] = e; m.ve_nbr[cur[a]++] = b;
      m.ve_edge[cur[b]] = e; m.ve_nbr[cur[b]++] = a;
    }
  }
  // vertex -> faces (ascending face id)
  m.vf_ptr.assign((size_t)V + 1, 0);
  for (size_t i = 0; i < 3 * (size_t)F; ++i) m.vf_ptr[m.faces[i] + 1]++;
  for (uint32_t v = 0; v < V; ++v) m.vf_ptr[v + 1] += m.vf_ptr[v];
  m.vf_face.resize(m.vf_ptr[V]);
  {
    std::vector<uint32_t> cur(m.vf_ptr.begin(), m.vf_ptr.end() - 1);
    for (uint32_t f = 0; f < F; ++f)
      for (int k = 0; k < 3; ++k) m.vf_face[cur[m.faces[3 * (size_t)f + k]]++] = f;
  }
}

// edge id between two vertices of face f (lvr2 getEdgeBetween, cvp:380-388, inflation:255-257)
inline uint32_t edgeBetweenInFace(const OrcMesh& m, uint32_t f, uint32_t a, uint32_t b) {
  const uint32_t* v = &m.faces[3 * (size_t)f];
  for (int k = 0; k < 3; ++k) {
    uint32_t p = v[k], q = v[(k + 1) % 3];
    if ((p == a && q == b) || (p == b && q == a)) return m.face_edges[3 * (size_t)f + k];
  }
  return 0xffffffffu;
}

// ---------------------------------------------------------------------------
// CVPMeshPlanner::waveFrontUpdate (default variant)  cvp_mesh_planner.cpp:369-556
// ---------------------------------------------------------------------------
struct CvpState {
  float* distances; uint32_t* predecessors; float* direction; int32_t* cutting_faces;
};

inline bool cvpWaveFrontUpdate(const OrcMesh& m, CvpState& s, const float* edge_weights,
                               uint32_t face, uint32_t v1, uint32_t v2, uint32_t v3) {
  const double u1 = s.distances[v1];                                   // :376
  const double u2 = s.distances[v2];
  const double u3 = s.distances[v3];
  const double c = edge_weights[edgeBetweenInFace(m, face, v1, v2)];   // :380-382
  const double c_sq = c * c;
  const double b = edge_weights[edgeBetweenInFace(m, face, v1, v3)];   // :384-386
  const double b_sq = b * b;
  const double a = edge_weights[edgeBetweenInFace(m, face, v2, v3)];   // :388-390
  const double a_sq = a * a;
  const double u1_sq = u1 * u1;
  const double u2_sq = u2 * u2;
  const double sx = (c_sq + u1_sq - u2_sq) / (2 * c);                  // :395
  const double sy = -sqrt(std::max(u1_sq - sx * sx, 0.0));             // :396
  const double p = (b_sq + c_sq - a_sq) / (2 * c);                     // :398
  const double hc = sqrt(std::max(b_sq - p * p, 0.0));                 // :399
  const double dy = hc - sy;
  const double dx = p - sx;
  const double u3tmp_sq = dx * dx + dy * dy;
  double u3tmp = sqrt(u3tmp_sq);                                       // :405
  if (u3tmp < u3) {                                                    // :411
    const double t0a = (a_sq + b_sq - c_sq) / (2 * a * b);             // :413
    const double t1a = (u3tmp_sq + b_sq - u1_sq) / (2 * u3tmp * b);
    const double t2a = (a_sq + u3tmp_sq - u2_sq) / (2 * a * u3tmp);
    if (std::fabs(t1a) > 1) {                                          // :418
      u3tmp = u1 + b;
      if (u3tmp < u3) {
        s.cutting_faces[v3] = (int32_t)face; s.predecessors[v3] = v1;
        s.distances[v3] = static_cast<float>(u3tmp); s.direction[v3] = 0;
        return true;
      }
      return false;
    } else if (std::fabs(t2a) > 1) {                                   // :437
      u3tmp = u2 + a;
      if (u3tmp < u3) {
        s.cutting_faces[v3] = (int32_t)face; s.predecessors[v3] = v2;
        s.distances[v3] = static_cast<float>(u3tmp); s.direction[v3] = 0;
        return true;
      }
      return false;
    }
    const double theta0 = acos(t0a);                                   // :456-458
    const double theta1 = acos(t1a);
    const double theta2 = acos(t2a);
    if (theta1 < theta0 && theta2 < theta0) {                          // :493
      s.cutting_faces[v3] = (int32_t)face;
      s.distances[v3] = static_cast<float>(u3tmp);
      if (theta1 < theta2) { s.predecessors[v3] = v1; s.direction[v3] = (float)theta1; }
      else { s.predecessors[v3] = v2; s.direction[v3] = (float)(-theta2); }
      return true;
    } else if (theta1 < theta2) {                                      // :518
      u3tmp = u1 + b;
      if (u3tmp < u3) {
        s.cutting_faces[v3] = (int32_t)face; s.predecessors[v3] = v1;
        s.distances[v3] = static_cast<float>(u3tmp); s.direction[v3] = 0;
        return true;
      }
      return false;
    } else {                                                           // :536
      u3tmp = u2 + a;
      if (u3tmp < u3) {
        s.cutting_faces[v3] = (int32_t)face; s.predecessors[v3] = v2;
        s.distances[v3] = static_cast<float>(u3tmp); s.direction[v3] = 0;
        return true;
      }
      return false;
    }
  }
  return false;
}

// ---------------------------------------------------------------------------
// InflationLayer::computeUpdateSethianMethod  inflation_layer.cpp:181-234
// (float throughout; literal conditions, including `sin` not `sin^2` at :195)
// ---------------------------------------------------------------------------
constexpr float INFLATION_EPSILON = 1e-9;  // `const float EPSILON = 1e-9;` mesh_layers/include/mesh_layers/inflation_layer.h:46

inline float sethianUpdate(const float d1, const float d2, const float a, const float b,
                           const float dot, const float F) {
  float t = FINF;
  float r_cos_angle = dot;
  float r_sin_angle = std::sqrt(1 - dot * dot);
  float u = d2 - d1;
  float f2 = a * a + b * b - 2 * a * b * r_cos_angle;
  float f1 = b * u * (a * r_cos_angle - b);
  float f0 = b * b * (u * u - F * F * a * a * r_sin_angle);
  float delta = f1 * f1 - f0 * f2;
  if (delta >= 0) {
    if (std::fabs(f2) > INFLATION_EPSILON) {
      t = (-f1 - std::sqrt(delta)) / f2;
      if (t < u || b * (t - u) / t < a * r_cos_angle || a / r_cos_angle < b * (t - u) / 2) {
        t = (-f1 + std::sqrt(delta)) / f2;
      } else {
        if (f1 != 0) t = -f0 / f1; else t = -FINF;
      }
    }
  } else {
    t = -FINF;
  }
  if (u < t && a * r_cos_angle < b * (t - u) / t && b * (t - u) / t < a / r_cos_angle) return t + d1;
  return std::min(b * F + d1, a * F + d2);
}

inline void vnormalize(float* v) {
  float l = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (l > 0) { v[0] /= l; v[1] /= l; v[2] /= l; }
}

// InflationLayer::waveFrontUpdate  inflation_layer.cpp:236-313
inline bool inflationWaveFrontUpdate(const OrcMesh& m, float* distances, float* vector_map /*3V or null*/,
                                     const float max_distance, const float* edge_weights,
                                     uint32_t face, uint32_t v1h, uint32_t v2h, uint32_t v3h) {
  const float u1 = distances[v1h];
  const float u2 = distances[v2h];
  const float u3 = distances[v3h];
  if (u3 == 0) return false;                                                        // :252
  const float c = edge_weights[edgeBetweenInFace(m, face, v1h, v2h)];
  const float c_sq = c * c;
  const float b = edge_weights[edgeBetweenInFace(m, face, v1h, v3h)];
  const float b_sq = b * b;
  const float a = edge_weights[edgeBetweenInFace(m, face, v2h, v3h)];
  const float a_sq = a * a;
  float dot = (a_sq + b_sq - c_sq) / (2 * a * b);                                   // :268
  float u3tmp = sethianUpdate(u1, u2, a, b, dot, 1.0f);
  if (!std::isfinite(u3tmp)) return false;                                          // :271
  const float d31 = u3tmp - u1;
  const float d32 = u3tmp - u2;
  if (vector_map && u1 == 0 && u2 == 0) {                                           // :277-295
    const float* p1 = &m.pos[3 * (size_t)v1h]; const float* p2 = &m.pos[3 * (size_t)v2h];
    const float* p3 = &m.pos[3 * (size_t)v3h];
    float dir[3];
    for (int k = 0; k < 3; ++k) dir[k] = (p3[k] - p2[k]) + (p3[k] - p1[k]);
    vnormalize(dir);
    for (uint32_t vh : {v1h, v2h, v3h}) {
      float* vm = &vector_map[3 * (size_t)vh];
      for (int k = 0; k < 3; ++k) vm[k] = vm[k] + dir[k];
      vnormalize(vm);
    }
  }
  if (u3tmp < u3) {                                                                 // :297
    distances[v3h] = u3tmp;
    if (vector_map && (u1 != 0 || u2 != 0)) {
      const float* va = &vector_map[3 * (size_t)v1h]; const float* vb = &vector_map[3 * (size_t)v2h];
      float out[3];
      for (int k = 0; k < 3; ++k) out[k] = va[k] * d31 + vb[k] * d32;
      vnormalize(out);
      for (int k = 0; k < 3; ++k) vector_map[3 * (size_t)v3h + k] = out[k];
    }
    return u1 <= max_distance && u2 <= max_distance;                                // :310
  }
  return false;
}

struct InflationConfig {   // mesh_layers/include/mesh_layers/inflation_layer.h:240-248 (doubles)
  double inscribed_radius, inflation_radius, lethal_value, inscribed_value, cost_scaling_factor;
};

// InflationLayer::fading  inflation_layer.cpp:315-339 (config members are double)
inline float fading(const InflationConfig& cfg, const float distance) {
  if (distance > cfg.inflation_radius) return 0;
  if (distance > cfg.inscribed_radius) {
    const float factor = exp(-1.0f * cfg.cost_scaling_factor * (distance - cfg.inscribed_radius));
    const float cost = cfg.inscribed_value * factor;
    return cost;
  }
  if (distance > 0) return cfg.inscribed_value;
  return cfg.lethal_value;
}

inline double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

}  // namespace

// debugging aid for the tests/tools: when set, orc_cvp records the pop sequence number of every vertex
static uint32_t* g_pop_index = nullptr;

extern "C" {

void orc_debug_set_pop_buffer(uint32_t* buf) { g_pop_index = buf; }

void* orc_mesh_create(uint32_t V, uint32_t F, const float* pos, const uint32_t* faces,
                      const uint32_t* edges /*nullable*/, uint32_t E) {
  OrcMesh* m = new OrcMesh();
  m->V = V; m->F = F;
  m->pos.assign(pos, pos + 3 * (size_t)V);
  m->faces.assign(faces, faces + 3 * (size_t)F);
  buildTopology(*m, edges, E);
  return m;
}
void orc_mesh_destroy(void* h) { delete (OrcMesh*)h; }
uint32_t orc_mesh_num_edges(void* h) { return ((OrcMesh*)h)->E; }
void orc_mesh_get_edges(void* h, uint32_t* out) {
  OrcMesh* m = (OrcMesh*)h; std::memcpy(out, m->edges.data(), sizeof(uint32_t) * 2 * (size_t)m->E);
}

// lvr2::calcVertexDistances as used for MeshMap::edge_distances (mesh_map.cpp:404-425):
// Euclidean length of every edge, float arithmetic (BaseVector<float>::distanceFrom).
void orc_edge_distances(void* h, float* out) {
  OrcMesh* m = (OrcMesh*)h;
  for (uint32_t e = 0; e < m->E; ++e) {
    const float* p = &m->pos[3 * (size_t)m->edges[2 * (size_t)e]];
    const float* q = &m->pos[3 * (size_t)m->edges[2 * (size_t)e + 1]];
    float dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
    out[e] = std::sqrt(dx * dx + dy * dy + dz * dz);
  }
}

// MeshMap::computeEdgeWeights  mesh_map.cpp:517-561 (formula :539-553; edge_cost_factor is double, mesh_map.h:516)
void orc_edge_weights(void* h, const float* vertex_costs, const float* edge_distances,
                      double edge_cost_factor, float* edge_weights) {
  OrcMesh* m = (OrcMesh*)h;
  for (uint32_t e = 0; e < m->E; ++e) {
    const float v1cost = vertex_costs[m->edges[2 * (size_t)e]];
    const float v2cost = vertex_costs[m->edges[2 * (size_t)e + 1]];
    if (std::isinf(v1cost) || std::isinf(v2cost)) {
      edge_weights[e] = FINF;
    } else {
      const float vertex_dist = edge_distances[e];
      const float edge_cost = vertex_dist * (v1cost + v2cost) / 2.0;
      edge_weights[e] = vertex_dist + edge_cost_factor * edge_cost;
    }
  }
}

// ---------------------------------------------------------------------------
// DijkstraMeshPlanner::dijkstra  dijkstra_mesh_planner.cpp:217-398 (loop :287-348)
//   seed_vertex  = reference "start_vertex" (nearest vertex to the navigation goal, :235)
//   robot_vertex = reference "goal_vertex"  (nearest vertex to the robot, :236); -1 = none
// returns the MBF outcome code (0 SUCCESS, 54 NO_PATH_FOUND); stats[0]=fixed_set_cnt,
// stats[1]=expanded vertices (reached the edge loop), stats[2]=propagation seconds.
// ---------------------------------------------------------------------------
uint32_t orc_dijkstra(void* h, const float* edge_weights, const float* vertex_costs,
                      const uint8_t* invalid, uint32_t seed_vertex, int64_t robot_vertex,
                      double cost_limit, double goal_dist_offset, int canonical_ties,
                      float* distances, uint32_t* predecessors, double* stats) {
  OrcMesh& m = *(OrcMesh*)h;
  const uint32_t V = m.V;
  if (robot_vertex >= 0 && (uint32_t)robot_vertex == seed_vertex) return 0;          // :252-255
  std::vector<uint8_t> fixed(V, 0);                                                  // :257
  for (uint32_t v = 0; v < V; ++v) { distances[v] = FINF; predecessors[v] = v; }     // :266-270
  Meap pq(V, canonical_ties != 0);
  distances[seed_vertex] = 0;                                                        // :276
  pq.insert(seed_vertex, 0);
  float goal_dist = FINF;                                                            // :279
  size_t fixed_set_cnt = 0, expanded = 0;
  const double t0 = now_s();
  while (!pq.isEmpty()) {                                                            // :287
    uint32_t cur = pq.popMin().key;
    fixed[cur] = 1;
    fixed_set_cnt++;
    if (robot_vertex >= 0 && cur == (uint32_t)robot_vertex)                          // :293-297
      goal_dist = distances[cur] + goal_dist_offset;
    if (distances[cur] > goal_dist) continue;                                        // :299
    if (vertex_costs[cur] > cost_limit) continue;                                    // :302
    expanded++;
    for (uint32_t k = m.ve_ptr[cur]; k < m.ve_ptr[cur + 1]; ++k) {                   // :320
      uint32_t vH = m.ve_nbr[k];
      if (fixed[vH]) continue;                                                       // :326
      if (invalid && invalid[vH]) continue;                                          // :328
      float tmp_cost = distances[cur] + edge_weights[m.ve_edge[k]];                  // :331
      if (tmp_cost < distances[vH]) {                                                // :332
        distances[vH] = tmp_cost;
        pq.insert(vH, tmp_cost);
        predecessors[vH] = cur;
      }
    }
  }
  const double t1 = now_s();
  if (stats) { stats[0] = (double)fixed_set_cnt; stats[1] = (double)expanded; stats[2] = t1 - t0; }
  if (robot_vertex >= 0 && predecessors[robot_vertex] == (uint32_t)robot_vertex) return 54;  // :358-362
  return 0;
}

// ---------------------------------------------------------------------------
// CVPMeshPlanner::waveFrontPropagation  cvp_mesh_planner.cpp:651-970
// (seeding :719-728, heap loop :747-886).  seed_face/seed_pos = reference
// "start_face"/"start" (the navigation goal, :673), robot_face = reference
// "goal_face" (-1 = none, full field).
// stats: [0]=fixed_set_cnt [1]=expanded pops [2]=seconds [3]=#waveFrontUpdate calls
//        [4]=#accepted updates [5]=#pops whose key < running max popped key (non-monotone)
//        [6]=max back-step magnitude
// ---------------------------------------------------------------------------
uint32_t orc_cvp(void* h, const float* edge_weights, const float* vertex_costs, const uint8_t* invalid,
                 uint32_t seed_face, const float* seed_pos, int64_t robot_face,
                 double cost_limit, double goal_dist_offset, int canonical_ties,
                 float* distances, uint32_t* predecessors, float* direction, int32_t* cutting_faces,
                 double* stats) {
  OrcMesh& m = *(OrcMesh*)h;
  const uint32_t V = m.V;
  std::vector<uint8_t> fixed(V, 0);                                                  // :702
  for (uint32_t v = 0; v < V; ++v) {                                                 // :710-714
    distances[v] = FINF; predecessors[v] = v; direction[v] = 0; cutting_faces[v] = -1;
  }
  CvpState st{distances, predecessors, direction, cutting_faces};
  Meap pq(V, canonical_ties != 0);
  for (int k = 0; k < 3; ++k) {                                                      // :719-728
    uint32_t vH = m.faces[3 * (size_t)seed_face + k];
    const float dx = seed_pos[0] - m.pos[3 * (size_t)vH], dy = seed_pos[1] - m.pos[3 * (size_t)vH + 1],
                dz = seed_pos[2] - m.pos[3 * (size_t)vH + 2];
    const float dist = std::sqrt(dx * dx + dy * dy + dz * dz);
    distances[vH] = dist;
    cutting_faces[vH] = (int32_t)seed_face;
    fixed[vH] = 1;
    pq.insert(vH, dist);
  }
  uint32_t goal_vertices[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu};
  if (robot_face >= 0) for (int k = 0; k < 3; ++k) goal_vertices[k] = m.faces[3 * (size_t)robot_face + k];
  float goal_dist = FINF;                                                            // :738
  size_t fixed_set_cnt = 0, expanded = 0, n_updates = 0, n_accept = 0, n_back = 0;
  double max_back = 0; float hi_water = 0;
  const double t0 = now_s();
  while (!pq.isEmpty()) {                                                            // :747
    uint32_t cur = pq.popMin().key;
    fixed[cur] = 1;                                                                  // :751
    if (g_pop_index) g_pop_index[cur] = (uint32_t)fixed_set_cnt;
    fixed_set_cnt++;
    if (distances[cur] < hi_water) { n_back++; max_back = std::max(max_back, (double)(hi_water - distances[cur])); }
    else hi_water = distances[cur];
    if (distances[cur] > goal_dist) continue;                                        // :754
    if (vertex_costs[cur] >= cost_limit) continue;                                   // :757
    if (invalid && invalid[cur]) continue;                                           // :760
    if (cur == goal_vertices[0] || cur == goal_vertices[1] || cur == goal_vertices[2]) {  // :763-771
      if (goal_dist == FINF && fixed[goal_vertices[0]] && fixed[goal_vertices[1]] && fixed[goal_vertices[2]])
        goal_dist = distances[cur] + goal_dist_offset;
    }
    expanded++;
    for (uint32_t k = m.vf_ptr[cur]; k < m.vf_ptr[cur + 1]; ++k) {                   // :778
      const uint32_t fh = m.vf_face[k];
      const uint32_t a = m.faces[3 * (size_t)fh], b = m.faces[3 * (size_t)fh + 1], c = m.faces[3 * (size_t)fh + 2];
      if (invalid && (invalid[a] || invalid[b] || invalid[c])) continue;             // :785
      if (fixed[a] && fixed[b] && fixed[c]) continue;                                // :790
      else if (fixed[a] && fixed[b] && !fixed[c]) {                                  // :798
        if (vertex_costs[c] >= cost_limit) continue;
        n_updates++;
        if (cvpWaveFrontUpdate(m, st, edge_weights, fh, a, b, c)) { pq.insert(c, distances[c]); n_accept++; }
      } else if (fixed[a] && !fixed[b] && fixed[c]) {                                // :821
        if (vertex_costs[b] >= cost_limit) continue;
        n_updates++;
        if (cvpWaveFrontUpdate(m, st, edge_weights, fh, c, a, b)) { pq.insert(b, distances[b]); n_accept++; }
      } else if (!fixed[a] && fixed[b] && fixed[c]) {                                // :844
        if (vertex_costs[a] >= cost_limit) continue;
        n_updates++;
        if (cvpWaveFrontUpdate(m, st, edge_weights, fh, b, c, a)) { pq.insert(a, distances[a]); n_accept++; }
      } else continue;                                                               // :867
    }
  }
  const double t1 = now_s();
  if (stats) {
    stats[0] = (double)fixed_set_cnt; stats[1] = (double)expanded; stats[2] = t1 - t0;
    stats[3] = (double)n_updates; stats[4] = (double)n_accept; stats[5] = (double)n_back; stats[6] = max_back;
  }
  if (robot_face >= 0) {                                                             // :902-918
    bool any = false;
    for (int k = 0; k < 3; ++k) if (goal_vertices[k] != predecessors[goal_vertices[k]]) { any = true; break; }
    if (!any && (uint32_t)robot_face != seed_face) return 54;
  }
  return 0;
}

// single call of CVPMeshPlanner::waveFrontUpdate on face `face` (for derived golden vectors)
int orc_cvp_wavefront_update(void* h, const float* edge_weights, uint32_t face, uint32_t v1, uint32_t v2, uint32_t v3,
                             float* distances, uint32_t* predecessors, float* direction, int32_t* cutting_faces) {
  CvpState st{distances, predecessors, direction, cutting_faces};
  return cvpWaveFrontUpdate(*(OrcMesh*)h, st, edge_weights, face, v1, v2, v3) ? 1 : 0;
}

// single call of InflationLayer::waveFrontUpdate (pinned by inflation_layer_test.cpp:62-76)
int orc_inflation_wavefront_update(void* h, float* distances, float* vector_map, float max_distance,
                                   const float* edge_weights, uint32_t face, uint32_t v1, uint32_t v2, uint32_t v3) {
  return inflationWaveFrontUpdate(*(OrcMesh*)h, distances, vector_map, max_distance, edge_weights, face, v1, v2, v3) ? 1 : 0;
}

float orc_fading(double inscribed_radius, double inflation_radius, double lethal_value, double inscribed_value,
                 double cost_scaling_factor, float distance) {
  InflationConfig cfg{inscribed_radius, inflation_radius, lethal_value, inscribed_value, cost_scaling_factor};
  return fading(cfg, distance);
}

float orc_sethian_update(float d1, float d2, float a, float b, float dot, float F) {
  return sethianUpdate(d1, d2, a, b, dot, F);
}

// ---------------------------------------------------------------------------
// InflationLayer::waveCostInflation  inflation_layer.cpp:341-491 (loop :407-478)
// lethals must be ascending (std::set iteration order, :397).  distances: +inf
// = "not in the sparse map".  cost_out: NaN = "not in the sparse map" (:484-490).
// stats: [0]=pops [1]=seconds [2]=update calls
// ---------------------------------------------------------------------------
void orc_inflation(void* h, const float* edge_distances, const uint8_t* invalid,
                   const uint32_t* lethals, uint32_t n_lethals,
                   double inscribed_radius, double inflation_radius, double lethal_value,
                   double inscribed_value, double cost_scaling_factor, int canonical_ties,
                   float* distances, float* cost_out, float* vector_out /*nullable 3V*/, double* stats) {
  OrcMesh& m = *(OrcMesh*)h;
  const uint32_t V = m.V;
  InflationConfig cfg{inscribed_radius, inflation_radius, lethal_value, inscribed_value, cost_scaling_factor};
  const float max_distance = (float)inflation_radius;   // double -> `const float&` parameter (:450, :240)
  std::vector<uint8_t> fixed(V, 0);
  for (uint32_t v = 0; v < V; ++v) distances[v] = FINF;
  if (vector_out) std::memset(vector_out, 0, sizeof(float) * 3 * (size_t)V);
  Meap pq(V, canonical_ties != 0);
  for (uint32_t i = 0; i < n_lethals; ++i) {                                         // :397-402
    uint32_t vH = lethals[i];
    distances[vH] = 0.0f; fixed[vH] = 1; pq.insert(vH, 0);
  }
  size_t pops = 0, calls = 0;
  const double t0 = now_s();
  while (!pq.isEmpty()) {                                                            // :407
    uint32_t cur = pq.popMin().key;
    pops++;
    if (cur >= V) continue;                                                          // :412
    if (invalid && invalid[cur]) continue;                                           // :417
    fixed[cur] = 1;                                                                  // :422
    for (uint32_t k = m.ve_ptr[cur]; k < m.ve_ptr[cur + 1]; ++k) {                   // :423 neighbours
      const uint32_t e = m.ve_edge[k];
      for (int side = 0; side < 2; ++side) {                                         // :427 both faces of the halfedge
        const int32_t fh = m.edge_faces[2 * (size_t)e + side];
        if (fh < 0) continue;
        const uint32_t a = m.faces[3 * (size_t)fh], b = m.faces[3 * (size_t)fh + 1], c = m.faces[3 * (size_t)fh + 2];
        if (fixed[a] && fixed[b] && fixed[c]) continue;                              // :443
        else if (fixed[a] && fixed[b] && !fixed[c]) {
          calls++;
          if (inflationWaveFrontUpdate(m, distances, vector_out, max_distance, edge_distances, fh, a, b, c)) pq.insert(c, distances[c]);
        } else if (fixed[a] && !fixed[b] && fixed[c]) {
          calls++;
          if (inflationWaveFrontUpdate(m, distances, vector_out, max_distance, edge_distances, fh, c, a, b)) pq.insert(b, distances[b]);
        } else if (!fixed[a] && fixed[b] && fixed[c]) {
          calls++;
          if (inflationWaveFrontUpdate(m, distances, vector_out, max_distance, edge_distances, fh, b, c, a)) pq.insert(a, distances[a]);
        } else continue;
      }
    }
  }
  const double t1 = now_s();
  for (uint32_t v = 0; v < V; ++v)                                                   // :482-490
    cost_out[v] = std::isinf(distances[v]) ? std::numeric_limits<float>::quiet_NaN() : fading(cfg, distances[v]);
  if (stats) { stats[0] = (double)pops; stats[1] = t1 - t0; stats[2] = (double)calls; }
}


// ---------------------------------------------------------------------------
// Geometric cost layers (mesh_layers/src/*_layer.cpp).  Steepness, Ridge, the Clearance cost mapping,
// the lethal rule (cost > threshold) and the Max combination are in the reference tree; height
// differences, roughness, border costs, normals and the radius neighbourhood are lvr2 functions
// (calcVertexHeightDifferences, calcVertexRoughness, calcBorderCosts, calcFaceNormals,
// calcVertexNormals, visitLocalVertexNeighborhood -- un-vendored, lvr2 @ main).  Their DEFINITIONS
// here are this repo's documented restatement (SURVEY.md 8c), not verifiable offline: PARITY UNPINNED.
//   face normal    = normalize(cross(p1 - p0, p2 - p0))
//   vertex normal  = normalize(sum of incident face normals, ascending face id)
//   neighbourhood  = stack traversal from v over mesh edges (CSR order); a not-yet-seen neighbour n is
//                    marked seen, and if |p_n - p_v| < radius it is visited and pushed; v itself is not visited
// ---------------------------------------------------------------------------
}  // extern "C"
// acos of a float, evaluated in double and rounded once.  The reference (roughness via lvr2, steepness_layer.cpp:165) calls
// its libm's float overload, whose last bit differs between libm versions; lethal sets are threshold tests on these
// values, so the oracle and the CUDA kernels both use the correctly rounded value (see kernels_layers.cuh, acos_f).
static inline float acosF(float x) { return (float)std::acos((double)x); }
static inline void vsub(const float* a, const float* b, float* o) { o[0] = a[0] - b[0]; o[1] = a[1] - b[1]; o[2] = a[2] - b[2]; }

extern "C" void orc_normals(void* h, float* face_normals /*3F*/, float* vertex_normals /*3V*/) {
  OrcMesh& m = *(OrcMesh*)h;
  for (uint32_t f = 0; f < m.F; ++f) {
    const float* p0 = &m.pos[3 * (size_t)m.faces[3 * (size_t)f]];
    const float* p1 = &m.pos[3 * (size_t)m.faces[3 * (size_t)f + 1]];
    const float* p2 = &m.pos[3 * (size_t)m.faces[3 * (size_t)f + 2]];
    float a[3], b[3], n[3];
    vsub(p1, p0, a); vsub(p2, p0, b);
    n[0] = a[1] * b[2] - a[2] * b[1]; n[1] = a[2] * b[0] - a[0] * b[2]; n[2] = a[0] * b[1] - a[1] * b[0];
    vnormalize(n);
    for (int k = 0; k < 3; ++k) face_normals[3 * (size_t)f + k] = n[k];
  }
  for (uint32_t v = 0; v < m.V; ++v) {
    float n[3] = {0, 0, 0};
    for (uint32_t k = m.vf_ptr[v]; k < m.vf_ptr[v + 1]; ++k)
      for (int c = 0; c < 3; ++c) n[c] = n[c] + face_normals[3 * (size_t)m.vf_face[k] + c];
    vnormalize(n);
    for (int c = 0; c < 3; ++c) vertex_normals[3 * (size_t)v + c] = n[c];
  }
}

struct OrcLayerParams {            // config structs at the end of mesh_layers/include/mesh_layers/*_layer.h
  double height_diff_threshold, height_diff_radius;      // 0.185, 0.3
  double roughness_threshold, roughness_radius;          // 0.3, 0.3
  double steepness_threshold;                            // 0.3
  double ridge_threshold, ridge_radius;                  // 0.3, 0.3
  double clearance_robot_height, clearance_height_inflation;  // 0.5, 0.3
  double border_threshold, border_cost;                  // 0.5, 1.0
};

template <class Visit>
static void visitNeighbourhood(const OrcMesh& m, uint32_t v, float radius, std::vector<uint32_t>& seen,
                               std::vector<uint32_t>& stack, Visit visit) {
  seen.clear(); stack.clear();
  seen.push_back(v); stack.push_back(v);
  const float* pv = &m.pos[3 * (size_t)v];
  while (!stack.empty()) {
    const uint32_t u = stack.back(); stack.pop_back();
    for (uint32_t k = m.ve_ptr[u]; k < m.ve_ptr[u + 1]; ++k) {
      const uint32_t n = m.ve_nbr[k];
      bool was = false;
      for (uint32_t s : seen) if (s == n) { was = true; break; }
      if (was) continue;
      seen.push_back(n);
      const float* pn = &m.pos[3 * (size_t)n];
      const float dx = pn[0] - pv[0], dy = pn[1] - pv[1], dz = pn[2] - pv[2];
      if (std::sqrt(dx * dx + dy * dy + dz * dz) < radius) { visit(n); stack.push_back(n); }
    }
  }
}

// costs: 6 arrays of V floats in the order height_diff, roughness, steepness, ridge, clearance, border;
// combined = MaxCombinationLayer (combination_layer.cpp:44-85); lethal_mask bit i = lethal in layer i
// (computeLethals: cost > threshold, e.g. height_diff_layer.cpp:67-79; clearance: clearance < robot_height,
// clearance_layer.cpp:79-83).  clearance may be null (= +inf everywhere: no ray hits, SURVEY.md H6).
extern "C" void orc_layers(void* h, const OrcLayerParams* P, const float* vertex_normals, const float* clearance,
                float* height_diff, float* roughness, float* steepness, float* ridge, float* clearance_cost,
                float* border, float* combined, uint8_t* lethal_mask) {
  OrcMesh& m = *(OrcMesh*)h;
  std::vector<uint32_t> seen, stack;
  std::vector<uint8_t> is_border(m.V, 0);
  for (uint32_t e = 0; e < m.E; ++e)
    if (m.edge_faces[2 * (size_t)e + 1] < 0) { is_border[m.edges[2 * (size_t)e]] = 1; is_border[m.edges[2 * (size_t)e + 1]] = 1; }
  for (uint32_t v = 0; v < m.V; ++v) {
    const float* pv = &m.pos[3 * (size_t)v];
    const float* nv = &vertex_normals[3 * (size_t)v];
    // height differences: max - min of z over the neighbourhood including v (lvr2::calcVertexHeightDifferences)
    float zmin = pv[2], zmax = pv[2];
    visitNeighbourhood(m, v, (float)P->height_diff_radius, seen, stack, [&](uint32_t n) {
      const float z = m.pos[3 * (size_t)n + 2];
      zmin = std::min(zmin, z); zmax = std::max(zmax, z);
    });
    const float hd = zmax - zmin;
    // roughness: mean angle between the vertex normal and the neighbours' normals (lvr2::calcVertexRoughness)
    float rsum = 0.0f; int rcnt = 0;
    visitNeighbourhood(m, v, (float)P->roughness_radius, seen, stack, [&](uint32_t n) {
      const float* nn = &vertex_normals[3 * (size_t)n];
      float dot = nv[0] * nn[0] + nv[1] * nn[1] + nv[2] * nn[2];
      dot = std::min(1.0f, std::max(-1.0f, dot));
      rsum = rsum + acosF(dot); rcnt++;
    });
    const float ro = rcnt ? rsum / (float)rcnt : 0.0f;
    // steepness (steepness_layer.cpp:165)
    const float st = acosF(nv[2]);
    // ridge (ridge_layer.cpp:155-184)
    float value = 0.0f; int num = 0;
    const float ref[3] = {pv[0] + nv[0], pv[1] + nv[1], pv[2] + nv[2]};
    visitNeighbourhood(m, v, (float)P->ridge_radius, seen, stack, [&](uint32_t n) {
      const float* pn = &m.pos[3 * (size_t)n]; const float* nn = &vertex_normals[3 * (size_t)n];
      const float cx = (pn[0] + nn[0]) - ref[0], cy = (pn[1] + nn[1]) - ref[1], cz = (pn[2] + nn[2]) - ref[2];
      value += std::sqrt(cx * cx + cy * cy + cz * cz);
      num++;
    });
    const float ri = num == 0 ? (float)(P->ridge_threshold + 0.1) : value / num;
    // clearance cost mapping (clearance_layer.cpp:77-96)
    const float cl = clearance ? clearance[v] : FINF;
    float cc; bool cl_lethal = false;
    const double inflated_height = P->clearance_robot_height + P->clearance_height_inflation;
    if (cl < P->clearance_robot_height) { cc = 1.0f; cl_lethal = true; }
    else if (cl < inflated_height) {
      const double diff = (cl - P->clearance_robot_height) / P->clearance_height_inflation;
      cc = (float)((cos(diff * M_PI) + 1.0) / 2.0);
    } else cc = 0.0f;
    // border (lvr2::calcBorderCosts)
    const float bo = is_border[v] ? (float)P->border_cost : 0.0f;
    height_diff[v] = hd; roughness[v] = ro; steepness[v] = st; ridge[v] = ri; clearance_cost[v] = cc; border[v] = bo;
    uint8_t mask = 0;
    if (hd > P->height_diff_threshold) mask |= 1;
    if (ro > P->roughness_threshold) mask |= 2;
    if (st > P->steepness_threshold) mask |= 4;
    if (ri > P->ridge_threshold) mask |= 8;
    if (cl_lethal) mask |= 16;
    if (bo > P->border_threshold) mask |= 32;
    lethal_mask[v] = mask;
    float c = 0.0f;                                         // MaxCombinationLayer default value 0
    c = std::max(c, hd); c = std::max(c, ro); c = std::max(c, st); c = std::max(c, ri); c = std::max(c, cc); c = std::max(c, bo);
    combined[v] = c;
  }
}



// ---------------------------------------------------------------------------
// DijkstraMeshPlanner::computeVectorMap  dijkstra_mesh_planner.cpp:189-209
// vector_map[v3] = normalize(p[pred[v3]] - p[v3]) for pred != self; NaN = "not in the sparse map".
// ---------------------------------------------------------------------------
extern "C" void orc_dijkstra_vector_map(void* h, const uint32_t* predecessors, float* vector_map /*3V*/) {
  OrcMesh& m = *(OrcMesh*)h;
  const float nan = std::numeric_limits<float>::quiet_NaN();
  for (uint32_t v3 = 0; v3 < m.V; ++v3) {
    float* o = &vector_map[3 * (size_t)v3];
    const uint32_t v1 = predecessors[v3];
    if (v1 == v3) { o[0] = o[1] = o[2] = nan; continue; }
    float d[3]; vsub(&m.pos[3 * (size_t)v1], &m.pos[3 * (size_t)v3], d);
    vnormalize(d);
    o[0] = d[0]; o[1] = d[1]; o[2] = d[2];
  }
}

// ---------------------------------------------------------------------------
// CVPMeshPlanner::computeVectorMap  cvp_mesh_planner.cpp:204-239
// vector_map[v3] = normalize(rotated(p[pred] - p[v3], axis = vertex_normal[v3], angle = direction[v3])), skipped if
// pred == self or no cutting face.  lvr2::BaseVector::rotated is un-vendored: restated as the Rodrigues rotation
// with sin/cos evaluated in double (the angle parameter is `const double&`) -- PARITY UNPINNED.
// ---------------------------------------------------------------------------
extern "C" void orc_cvp_vector_map(void* h, const float* vertex_normals, const uint32_t* predecessors, const float* direction,
                                   const int32_t* cutting_faces, float* vector_map /*3V*/) {
  OrcMesh& m = *(OrcMesh*)h;
  const float nan = std::numeric_limits<float>::quiet_NaN();
  for (uint32_t v3 = 0; v3 < m.V; ++v3) {
    float* o = &vector_map[3 * (size_t)v3];
    const uint32_t v1 = predecessors[v3];
    if (v1 == v3 || cutting_faces[v3] < 0) { o[0] = o[1] = o[2] = nan; continue; }     // :218, :224
    float v[3]; vsub(&m.pos[3 * (size_t)v1], &m.pos[3 * (size_t)v3], v);
    const float* n = &vertex_normals[3 * (size_t)v3];
    const double alpha = direction[v3];
    const float sina = (float)sin(alpha), cosa = (float)cos(alpha);
    const float ndotv = n[0] * v[0] + n[1] * v[1] + n[2] * v[2];
    const float cx = n[1] * v[2] - n[2] * v[1], cy = n[2] * v[0] - n[0] * v[2], cz = n[0] * v[1] - n[1] * v[0];
    float r[3] = {v[0] * cosa + cx * sina + n[0] * ndotv * (1.0f - cosa),
                  v[1] * cosa + cy * sina + n[1] * ndotv * (1.0f - cosa),
                  v[2] * cosa + cz * sina + n[2] * ndotv * (1.0f - cosa)};
    vnormalize(r);
    o[0] = r[0]; o[1] = r[1]; o[2] = r[2];
  }
}

// ---------------------------------------------------------------------------
// Vector-field back-tracking: CVPMeshPlanner::waveFrontPropagation cvp_mesh_planner.cpp:920-951 over
// MeshMap::meshAhead mesh_map.cpp:1070-1108, searchNeighbourFaces :999-1068, directionAtPosition :625-650 and
// projectedBarycentricCoords util.cpp:313-347.  Layer vector fields (AbstractLayer::vectorAt) contribute zero
// (no layer with a repulsive field is built yet -- SURVEY f4).  lvr2's getFacesOfVertex order is un-vendored:
// ascending face id here -- PARITY UNPINNED for the (rare) case of two faces both passing the inside test.
// vector_map: 3V floats, NaN row = no entry.  The walk starts at the robot (the wave's `goal`) and ends at the
// wave's seed (`start`); points are written in walk order.  Returns 0 SUCCESS / 54 NO_PATH_FOUND / -1 cap hit.
// ---------------------------------------------------------------------------
namespace {
struct V3 { float x, y, z; };
inline V3 sub3(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline V3 cross3(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
inline float dot3(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline V3 P(const OrcMesh& m, uint32_t v) { return {m.pos[3 * (size_t)v], m.pos[3 * (size_t)v + 1], m.pos[3 * (size_t)v + 2]}; }

// util.cpp:313-347
inline bool projectedBarycentricCoords(V3 p, V3 a, V3 b, V3 c, float bary[3], float& dist) {
  const V3 u = sub3(b, a), v = sub3(c, a), w = sub3(p, a), n = cross3(u, v);
  const float oneOver4ASquared = (float)(1.0 / (double)dot3(n, n));
  const float gamma = dot3(cross3(u, w), n) * oneOver4ASquared;
  const float beta = dot3(cross3(w, v), n) * oneOver4ASquared;
  const float alpha = 1 - gamma - beta;
  bary[0] = alpha; bary[1] = beta; bary[2] = gamma;
  dist = dot3(n, w) / std::sqrt(dot3(n, n));
  const float EPSILON = 0.01f;
  return (0 - EPSILON <= alpha) && (alpha <= 1 + EPSILON) && (0 - EPSILON <= beta) && (beta <= 1 + EPSILON) &&
         (0 - EPSILON <= gamma) && (gamma <= 1 + EPSILON);
}

// mesh_map.cpp:999-1068
inline bool searchNeighbourFaces(const OrcMesh& m, V3 pos, uint32_t face, float max_radius, float max_dist, uint32_t& face_out,
                                 float bary[3]) {
  std::vector<uint32_t> possible{face};
  const uint32_t* fv = &m.faces[3 * (size_t)face];
  V3 center{0, 0, 0};
  for (int k = 0; k < 3; ++k) { const V3 q = P(m, fv[k]); center = {center.x + q.x, center.y + q.y, center.z + q.z}; }
  center = {center.x / 3, center.y / 3, center.z / 3};
  float vertex_center_max = 0;
  for (int k = 0; k < 3; ++k) { const V3 d = sub3(P(m, fv[k]), center); vertex_center_max = std::max(vertex_center_max, std::sqrt(dot3(d, d))); }
  const float ext_radius = max_radius + vertex_center_max;
  const float max_radius_sq = ext_radius * ext_radius;
  std::unordered_set<uint32_t> in_list{face};
  for (size_t it = 0; it < possible.size(); ++it) {
    const uint32_t* t = &m.faces[3 * (size_t)possible[it]];
    float dist;
    if (projectedBarycentricCoords(pos, P(m, t[0]), P(m, t[1]), P(m, t[2]), bary, dist) && std::fabs(dist) < max_dist) {
      face_out = possible[it];
      return true;
    }
    for (int k = 0; k < 3; ++k) {
      const V3 d = sub3(center, P(m, t[k]));
      if (dot3(d, d) < max_radius_sq)
        for (uint32_t j = m.vf_ptr[t[k]]; j < m.vf_ptr[t[k] + 1]; ++j)
          if (in_list.insert(m.vf_face[j]).second) possible.push_back(m.vf_face[j]);
    }
  }
  return false;
}

// mesh_map.cpp:1070-1108 (+ directionAtPosition :625-650)
// InflationLayer::vectorAt(vertices, barycentric_coords)  inflation_layer.cpp:493-521.  lvr2's BaseVector<float> is
// un-vendored: `vec * double` is taken as a float scale; a face vertex without a distance entry (the reference would
// panic inside lvr2's DenseVertexMap::operator[]) yields the zero vector.  PARITY UNPINNED.
struct RepulsiveField {
  const float* distances;      // V, +inf = no entry
  const float* vectors;        // 3V, zero = no entry
  double inscribed_radius, inflation_radius, lethal_value, inscribed_value;
};
inline V3 inflationVectorAt(const RepulsiveField& L, const uint32_t* t, const float* bary) {
  const float d0 = L.distances[t[0]], d1 = L.distances[t[1]], d2 = L.distances[t[2]];
  if (!std::isfinite(d0) || !std::isfinite(d1) || !std::isfinite(d2)) return V3{0, 0, 0};
  const float distance = d0 * bary[0] + d1 * bary[1] + d2 * bary[2];                 // util.h:179-184
  if (distance > L.inflation_radius) return V3{0, 0, 0};
  const float* a = &L.vectors[3 * (size_t)t[0]]; const float* b = &L.vectors[3 * (size_t)t[1]]; const float* c = &L.vectors[3 * (size_t)t[2]];
  V3 v{a[0] * bary[0] + b[0] * bary[1] + c[0] * bary[2], a[1] * bary[0] + b[1] * bary[1] + c[1] * bary[2],
       a[2] * bary[0] + b[2] * bary[1] + c[2] * bary[2]};
  if (distance > L.inscribed_radius) {                                               // :505-511
    const float alpha = (std::sqrt(distance) - L.inscribed_radius) / (L.inflation_radius - L.inscribed_radius) * M_PI;
    const float s1 = (float)L.inscribed_value, s2 = std::cos(alpha) + 1, s3 = 2.0f;
    return V3{v.x * s1 * s2 / s3, v.y * s1 * s2 / s3, v.z * s1 * s2 / s3};
  }
  const float s = distance > 0 ? (float)L.inscribed_value : (float)L.lethal_value;   // :514-520
  return V3{v.x * s, v.y * s, v.z * s};
}

inline bool meshAhead(const OrcMesh& m, const float* vector_map, V3& pos, uint32_t& face, float step_size,
                      const RepulsiveField* layer = nullptr) {
  float bary[3], dist;
  const uint32_t* t = &m.faces[3 * (size_t)face];
  if (projectedBarycentricCoords(pos, P(m, t[0]), P(m, t[1]), P(m, t[2]), bary, dist)) {
  } else if (searchNeighbourFaces(m, pos, face, step_size, 0.4f, face, bary)) {
    t = &m.faces[3 * (size_t)face];
    const V3 a = P(m, t[0]), b = P(m, t[1]), c = P(m, t[2]);      // linearCombineBarycentricCoords util.h:179-184
    pos = {a.x * bary[0] + b.x * bary[1] + c.x * bary[2], a.y * bary[0] + b.y * bary[1] + c.y * bary[2],
           a.z * bary[0] + b.z * bary[1] + c.z * bary[2]};
  } else {
    return false;
  }
  bool any = false;
  V3 vec{0, 0, 0};
  for (int k = 0; k < 3; ++k) {
    const float* e = &vector_map[3 * (size_t)t[k]];
    if (std::isnan(e[0])) continue;
    any = true;
    vec = {vec.x + e[0] * bary[k], vec.y + e[1] * bary[k], vec.z + e[2] * bary[k]};
  }
  if (!any || !(std::isfinite(vec.x) && std::isfinite(vec.y) && std::isfinite(vec.z))) return false;
  float d[3] = {vec.x, vec.y, vec.z};
  vnormalize(d);          // opt_dir.normalized()
  if (layer) {            // dir += layer->vectorAt(handels, bary_coords) for every layer (mesh_map.cpp:1097-1102)
    const V3 lv = inflationVectorAt(*layer, t, bary);
    d[0] += lv.x; d[1] += lv.y; d[2] += lv.z;
  }
  vnormalize(d);          // dir.normalize()
  pos = {pos.x + d[0] * step_size, pos.y + d[1] * step_size, pos.z + d[2] * step_size};
  return true;
}
}  // namespace

static int32_t backtrackImpl(const OrcMesh& m, const float* vector_map, const float start[3], uint32_t start_face, const float goal[3],
                             uint32_t goal_face, double step_width, uint32_t max_points, float* path_pos, uint32_t* path_face,
                             uint32_t* n_points, const RepulsiveField* layer);
extern "C" int32_t orc_cvp_backtrack(void* h, const float* vector_map, const float start[3], uint32_t start_face, const float goal[3],
                                     uint32_t goal_face, double step_width, uint32_t max_points, float* path_pos, uint32_t* path_face,
                                     uint32_t* n_points) {
  return backtrackImpl(*(OrcMesh*)h, vector_map, start, start_face, goal, goal_face, step_width, max_points, path_pos, path_face, n_points, nullptr);
}
// same walk with the InflationLayer's repulsive field added in meshAhead (mesh_map.cpp:1097-1102)
extern "C" int32_t orc_cvp_backtrack_repulsive(void* h, const float* vector_map, const float start[3], uint32_t start_face,
                                               const float goal[3], uint32_t goal_face, double step_width, uint32_t max_points,
                                               float* path_pos, uint32_t* path_face, uint32_t* n_points,
                                               const float* infl_distances, const float* infl_vectors, double inscribed_radius,
                                               double inflation_radius, double lethal_value, double inscribed_value) {
  RepulsiveField L{infl_distances, infl_vectors, inscribed_radius, inflation_radius, lethal_value, inscribed_value};
  return backtrackImpl(*(OrcMesh*)h, vector_map, start, start_face, goal, goal_face, step_width, max_points, path_pos, path_face, n_points, &L);
}
// InflationLayer::vectorAt for n (face, barycentric) samples
extern "C" void orc_inflation_vector_at(void* h, uint32_t n, const uint32_t* faces_q, const float* bary, const float* infl_distances,
                                        const float* infl_vectors, double inscribed_radius, double inflation_radius,
                                        double lethal_value, double inscribed_value, float* out /*3n*/) {
  const OrcMesh& m = *(OrcMesh*)h;
  RepulsiveField L{infl_distances, infl_vectors, inscribed_radius, inflation_radius, lethal_value, inscribed_value};
  for (uint32_t q = 0; q < n; ++q) {
    const V3 v = inflationVectorAt(L, &m.faces[3 * (size_t)faces_q[q]], &bary[3 * (size_t)q]);
    out[3 * (size_t)q] = v.x; out[3 * (size_t)q + 1] = v.y; out[3 * (size_t)q + 2] = v.z;
  }
}
static int32_t backtrackImpl(const OrcMesh& m, const float* vector_map, const float start[3], uint32_t start_face, const float goal[3],
                             uint32_t goal_face, double step_width, uint32_t max_points, float* path_pos, uint32_t* path_face,
                             uint32_t* n_points, const RepulsiveField* layer) {
  uint32_t n = 0;
  auto push = [&](V3 p, uint32_t f) { if (n < max_points) { path_pos[3 * n] = p.x; path_pos[3 * n + 1] = p.y; path_pos[3 * n + 2] = p.z; path_face[n] = f; } ++n; };
  uint32_t current_face = goal_face;                                                    // :920
  V3 current_pos{goal[0], goal[1], goal[2]};
  const V3 st{start[0], start[1], start[2]};
  push(current_pos, current_face);
  const float sw = (float)step_width;
  for (;;) {
    const V3 d = sub3(current_pos, st);
    if (!((double)dot3(d, d) > step_width)) break;                                      // :925 distance2 vs step_width
    if (n + 1 >= max_points) { *n_points = n; return -1; }
    if (!meshAhead(m, vector_map, current_pos, current_face, sw, layer)) { *n_points = n; return 54; }   // :938-941
    push(current_pos, current_face);
  }
  push(st, start_face);                                                                 // :951
  *n_points = n;
  return 0;
}

// ---------------------------------------------------------------------------
// Localisation: MeshMap::getNearestVertexHandle mesh_map.cpp:1161-1174 (nanoflann 1-NN, L2_Simple: squared
// distance accumulated x, y, z in float; un-vendored -> exhaustive scan, ties to the lowest vertex id, PARITY
// UNPINNED for exact ties) and MeshMap::searchContainingFace mesh_map.cpp:1120-1159 (faces of the nearest vertex,
// ascending face id; the one with the lowest SIGNED plane distance among those passing the inside test; max_dist
// is not consulted by the reference).  face = -1: none.
// ---------------------------------------------------------------------------
extern "C" void orc_locate(void* h, uint32_t n, const float* points, uint32_t* nearest_vertex, int32_t* face, float* bary /*3n*/) {
  const OrcMesh& m = *(OrcMesh*)h;
  for (uint32_t q = 0; q < n; ++q) {
    const V3 p{points[3 * (size_t)q], points[3 * (size_t)q + 1], points[3 * (size_t)q + 2]};
    uint32_t best = 0; float bd = std::numeric_limits<float>::infinity();
    for (uint32_t v = 0; v < m.V; ++v) {
      const float dx = p.x - m.pos[3 * (size_t)v], dy = p.y - m.pos[3 * (size_t)v + 1], dz = p.z - m.pos[3 * (size_t)v + 2];
      const float d = dx * dx + dy * dy + dz * dz;
      if (d < bd) { bd = d; best = v; }
    }
    nearest_vertex[q] = best;
    float lowest = std::numeric_limits<float>::max();
    int32_t bf = -1; float bb[3] = {0, 0, 0};
    for (uint32_t k = m.vf_ptr[best]; k < m.vf_ptr[best + 1]; ++k) {
      const uint32_t f = m.vf_face[k];
      const uint32_t* t = &m.faces[3 * (size_t)f];
      float cb[3], dist = 0;
      if (projectedBarycentricCoords(p, P(m, t[0]), P(m, t[1]), P(m, t[2]), cb, dist) && dist < lowest) {
        lowest = dist; bf = (int32_t)f; bb[0] = cb[0]; bb[1] = cb[1]; bb[2] = cb[2];
      }
    }
    face[q] = bf;
    if (bary) { bary[3 * (size_t)q] = bb[0]; bary[3 * (size_t)q + 1] = bb[1]; bary[3 * (size_t)q + 2] = bb[2]; }
  }
}

// ---------------------------------------------------------------------------
// Incremental updates: the sensor-rate callers of the hot path (SURVEY.md 3.4 / 8f3).  NaN = "no entry in the sparse
// lvr2 map"; `changed` plays the std::set<VertexHandle> (ascending, unique).
// ---------------------------------------------------------------------------
// MeshMap::layerChanged  mesh_map.cpp:455-492, the vertex-cost part :478-487:
//   vertex_costs.insert(vH, cost_map.get(vH).value_or(default_value)) for vH in changes
extern "C" void orc_layer_changed(const float* layer_costs, float default_value, const uint32_t* changed, uint32_t n,
                                  float* vertex_costs) {
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t vH = changed[i];
    vertex_costs[vH] = std::isnan(layer_costs[vH]) ? default_value : layer_costs[vH];
  }
}

// MeshMap::updateEdgeWeights  mesh_map.cpp:563-618: only the edges incident to a changed vertex are recomputed, and
// NOTHING is recomputed when edge_cost_factor == 0 (:568-572) -- unlike computeEdgeWeights, an endpoint cost that
// became +inf then leaves the old weight in place.
extern "C" void orc_update_edge_weights(void* h, const float* vertex_costs, const float* edge_distances, double edge_cost_factor,
                                        const uint32_t* changed, uint32_t n, float* edge_weights) {
  OrcMesh* m = (OrcMesh*)h;
  if (0 == edge_cost_factor) return;                                                 // :568
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t changedH = changed[i];
    for (uint32_t k = m->ve_ptr[changedH]; k < m->ve_ptr[changedH + 1]; ++k) {       // getEdgesOfVertex :580
      const uint32_t eH = m->ve_edge[k];
      const float v1cost = vertex_costs[m->edges[2 * (size_t)eH]];
      const float v2cost = vertex_costs[m->edges[2 * (size_t)eH + 1]];
      if (std::isinf(v1cost) || std::isinf(v2cost)) {                                // :598
        edge_weights[eH] = FINF;
      } else {
        const float vertex_dist = edge_distances[eH];
        const float edge_cost = vertex_dist * (v1cost + v2cost) / 2.0;               // :609
        edge_weights[eH] = vertex_dist + edge_cost_factor * edge_cost;               // :611
      }
    }
  }
}

// MaxCombinationLayer::onInputChanged  combination_layer.cpp:87-147: for every changed vertex
//   cost = max over the input layers of (value or the layer's default), starting from 0 (:109-118);
//   lethal = the vertex is in the lethal set of any input (:122-139).
extern "C" void orc_max_combination_update(uint32_t n_layers, const float* const* layer_costs, const float* defaults,
                                           const uint8_t* const* layer_lethals, const uint32_t* changed, uint32_t n,
                                           float* costs, uint8_t* lethals) {
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t v = changed[i];
    float cost = 0;
    for (uint32_t l = 0; l < n_layers; ++l) {
      const float tmp = std::isnan(layer_costs[l][v]) ? defaults[l] : layer_costs[l][v];
      cost = std::max(tmp, cost);
    }
    costs[v] = cost;
  }
  if (lethals)
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t v = changed[i];
      bool lethal = false;
      for (uint32_t l = 0; l < n_layers; ++l) lethal = lethal || (layer_lethals[l] && layer_lethals[l][v]);
      lethals[v] = lethal ? 1 : 0;
    }
}

// AvgCombinationLayer::onInputChanged  combination_layer.cpp:250-302 (== computeLayer :185-248 on a costs_ map that still
// holds its initial default 0, :177-181): cost = sum over the input layers, in order, of combinationWeight * (value or
// default), float accumulation; lethal = the vertex is in the lethal set of any input.
extern "C" void orc_avg_combination_update(uint32_t n_layers, const float* const* layer_costs, const float* defaults,
                                           const float* weights, const uint8_t* const* layer_lethals, const uint32_t* changed,
                                           uint32_t n, float* costs, uint8_t* lethals) {
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t v = changed[i];
    float cost = 0;
    for (uint32_t l = 0; l < n_layers; ++l)
      cost += weights[l] * (std::isnan(layer_costs[l][v]) ? defaults[l] : layer_costs[l][v]);      // :269
    costs[v] = cost;
  }
  if (lethals)
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t v = changed[i];
      bool lethal = false;
      for (uint32_t l = 0; l < n_layers; ++l) lethal = lethal || (layer_lethals[l] && layer_lethals[l][v]);
      lethals[v] = lethal ? 1 : 0;
    }
}

// InflationLayer::onInputChanged  inflation_layer.cpp:154-164: the update set handed to notifyChange is the union of the
// keys of the new and of the previous riskiness map (std::set: ascending).  Returns its size.
extern "C" uint32_t orc_inflation_update_set(uint32_t V, const float* new_costs, const float* old_costs, uint32_t* out) {
  uint32_t n = 0;
  for (uint32_t v = 0; v < V; ++v)
    if (!std::isnan(new_costs[v]) || (old_costs && !std::isnan(old_costs[v]))) out[n++] = v;
  return n;
}

// ============================================================================
// Ray casting against the map (MeshMap::raycaster(), mesh_map.h:318; built at mesh_map.cpp:317-321 as
// lvr2::EmbreeRaycaster / lvr2::BVHRaycaster), ObstacleLayer::processPointCloud (obstacle_layer.cpp:215-296) and
// lvr2::calcNormalClearance (called at clearance_layer.cpp:161).
//
// PARITY UNPINNED: the ray/triangle arithmetic lives in lvr2 / Embree (un-vendored, source_dependencies.yaml:4-7) and the
// reference holds no test or golden vector for it.  Stated here and followed by the GPU kernels:
//   * a ray (o, d) meets a triangle (a, b, c) by the two-sided Moeller-Trumbore test in float, evaluated in the order written
//     in ray_triangle() below, and only inside the triangle's bounding box grown by eps = 1e-5f * max |coordinate| of the map
//     (box_span(): per-axis slabs; entry tn clamped at 0, exit tf; the hit needs tn <= t <= tf);
//   * of several hits the smallest t wins, ties go to the smallest face id;  dist = t (d is a unit vector at every call site),
//     point = o + d * t.
// This is a brute-force loop over all faces: the acceleration structure of the product must not change any result.
// ============================================================================
namespace {
struct OrcBox { float lo[3], hi[3]; };
inline bool box_span(const float o[3], const float d[3], const OrcBox& b, float& tn, float& tf) {
  tn = 0.0f; tf = FINF;
  for (int k = 0; k < 3; ++k) {
    if (!(std::fabs(d[k]) >= 1e-20f)) {
      if (o[k] < b.lo[k] || o[k] > b.hi[k]) return false;
    } else {
      const float inv = 1.0f / d[k];
      const float t1 = (b.lo[k] - o[k]) * inv, t2 = (b.hi[k] - o[k]) * inv;
      tn = std::fmax(tn, std::fmin(t1, t2));
      tf = std::fmin(tf, std::fmax(t1, t2));
    }
  }
  return tn <= tf;
}
inline float map_eps(const OrcMesh& m) {
  float mx = 0.0f;
  for (float x : m.pos) mx = std::fmax(mx, std::fabs(x));
  const float e = 1e-5f * mx;
  return e > 0.0f ? e : 1e-30f;
}
inline OrcBox tri_box(const OrcMesh& m, uint32_t f, float eps) {
  OrcBox b;
  const float* A = &m.pos[3 * (size_t)m.faces[3 * (size_t)f]];
  const float* B = &m.pos[3 * (size_t)m.faces[3 * (size_t)f + 1]];
  const float* Cc = &m.pos[3 * (size_t)m.faces[3 * (size_t)f + 2]];
  for (int k = 0; k < 3; ++k) {
    b.lo[k] = std::fmin(std::fmin(A[k], B[k]), Cc[k]) - eps;
    b.hi[k] = std::fmax(std::fmax(A[k], B[k]), Cc[k]) + eps;
  }
  return b;
}
inline bool ray_triangle(const float o[3], const float d[3], const float* a, const float* b, const float* c, float& t) {
  const float e1x = b[0] - a[0], e1y = b[1] - a[1], e1z = b[2] - a[2];
  const float e2x = c[0] - a[0], e2y = c[1] - a[1], e2z = c[2] - a[2];
  const float px = d[1] * e2z - d[2] * e2y, py = d[2] * e2x - d[0] * e2z, pz = d[0] * e2y - d[1] * e2x;
  const float det = (e1x * px + e1y * py) + e1z * pz;
  if (det == 0.0f) return false;
  const float inv = 1.0f / det;
  const float sx = o[0] - a[0], sy = o[1] - a[1], sz = o[2] - a[2];
  const float u = ((sx * px + sy * py) + sz * pz) * inv;
  if (!(u >= 0.0f && u <= 1.0f)) return false;
  const float qx = sy * e1z - sz * e1y, qy = sz * e1x - sx * e1z, qz = sx * e1y - sy * e1x;
  const float v = ((d[0] * qx + d[1] * qy) + d[2] * qz) * inv;
  if (!(v >= 0.0f && u + v <= 1.0f)) return false;
  t = ((e2x * qx + e2y * qy) + e2z * qz) * inv;
  return t >= 0.0f;
}
// nearest hit of one ray; skip_vertex: faces with this corner are ignored (UINT32_MAX = none)
inline bool cast_one(const OrcMesh& m, float eps, const float o[3], const float d[3], uint32_t skip_vertex, float& best_t, uint32_t& best_f) {
  bool any = false;
  for (uint32_t f = 0; f < m.F; ++f) {
    const uint32_t* fv = &m.faces[3 * (size_t)f];
    if (fv[0] == skip_vertex || fv[1] == skip_vertex || fv[2] == skip_vertex) continue;
    float tn, tf, t;
    if (!box_span(o, d, tri_box(m, f, eps), tn, tf)) continue;
    if (!ray_triangle(o, d, &m.pos[3 * (size_t)fv[0]], &m.pos[3 * (size_t)fv[1]], &m.pos[3 * (size_t)fv[2]], t)) continue;
    if (!(t >= tn && t <= tf)) continue;
    if (!any || t < best_t) { any = true; best_t = t; best_f = f; }       // ascending f: ties keep the smallest face id
  }
  return any;
}
}  // namespace

// lvr2::RaycasterBase::castRays as used at obstacle_layer.cpp:239: per ray hit flag, distance, face id, hit point.
// dir_stride 0: one direction for all rays (obstacle_layer.cpp:229), 3: one per ray.
extern "C" void orc_cast_rays(void* h, uint32_t n, const float* origins, const float* dirs, uint32_t dir_stride,
                              uint8_t* hit, float* dist, uint32_t* face, float* point) {
  const OrcMesh& m = *(const OrcMesh*)h;
  const float eps = map_eps(m);
  for (uint32_t i = 0; i < n; ++i) {
    const float* o = origins + 3 * (size_t)i; const float* d = dirs + (size_t)dir_stride * i;
    float t = 0; uint32_t f = 0;
    const bool any = cast_one(m, eps, o, d, 0xffffffffu, t, f);
    hit[i] = any ? 1 : 0;
    dist[i] = any ? t : FINF; face[i] = any ? f : 0xffffffffu;
    for (int k = 0; k < 3; ++k) point[3 * (size_t)i + k] = any ? o[k] + d[k] * t : std::numeric_limits<float>::quiet_NaN();
  }
}

// ObstacleLayer::processPointCloud  obstacle_layer.cpp:215-296.  points: the cloud in the sensor frame; tf: the 3x4 row-major
// [R|t] of the message frame -> map frame transform (:176-180; the caller expands its quaternion); axis: down_axis already
// rotated into the map frame (:183-205).  Points with |p| <= max_obstacle_dist are transformed (:221-226), one ray each along
// axis (:229-239); a hit no further than robot_height makes the three vertices of the hit face lethal (:245-256).
// lethal_mask (in: the previous lethal set, out: the new one) and changed_mask (symmetric difference, :268-273) are V bytes.
extern "C" void orc_obstacle_update(void* h, uint32_t n, const float* points, const float* tf, const float* axis,
                                    double max_obstacle_dist, double robot_height, uint8_t* lethal_mask, uint8_t* changed_mask) {
  const OrcMesh& m = *(const OrcMesh*)h;
  const float eps = map_eps(m);
  std::vector<uint8_t> now(m.V, 0);
  for (uint32_t i = 0; i < n; ++i) {
    const float x = points[3 * (size_t)i], y = points[3 * (size_t)i + 1], z = points[3 * (size_t)i + 2];
    const float norm = std::sqrt((x * x + y * y) + z * z);
    if (!((double)norm <= max_obstacle_dist)) continue;
    float o[3];
    for (int r = 0; r < 3; ++r) o[r] = ((tf[4 * r] * x + tf[4 * r + 1] * y) + tf[4 * r + 2] * z) + tf[4 * r + 3];
    float t = 0; uint32_t f = 0;
    if (cast_one(m, eps, o, axis, 0xffffffffu, t, f) && (double)t <= robot_height)
      for (int k = 0; k < 3; ++k) now[m.faces[3 * (size_t)f + k]] = 1;
  }
  for (uint32_t v = 0; v < m.V; ++v) { changed_mask[v] = now[v] != lethal_mask[v]; lethal_mask[v] = now[v]; }
}

// lvr2::calcNormalClearance (clearance_layer.cpp:161): the free space above a vertex = distance from the vertex along its
// normal to the first face that is not incident to it; +inf when nothing is hit or the normal is degenerate.
extern "C" void orc_normal_clearance(void* h, const float* vertex_normals, float* clearance) {
  const OrcMesh& m = *(const OrcMesh*)h;
  const float eps = map_eps(m);
  for (uint32_t v = 0; v < m.V; ++v) {
    const float* d = vertex_normals + 3 * (size_t)v;
    float t = 0; uint32_t f = 0;
    const bool ok = ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) > 0.0f;
    clearance[v] = (ok && cast_one(m, eps, &m.pos[3 * (size_t)v], d, v, t, f)) ? t : FINF;
  }
}
