// ROS-free C++ host mirror of the reference's plugin interface for the hot path, over the C ABI
// (include/meshnav_b200.h).  Same names, argument meaning and outcome codes as
//   mbf_mesh_core::MeshPlanner            mbf_mesh_core/include/mbf_mesh_core/mesh_planner.h:50-92
//   dijkstra_mesh_planner::DijkstraMeshPlanner   dijkstra_mesh_planner/src/dijkstra_mesh_planner.cpp
//   cvp_mesh_planner::CVPMeshPlanner             cvp_mesh_planner/src/cvp_mesh_planner.cpp
//   mesh_layers::InflationLayer                  mesh_layers/src/inflation_layer.cpp
// with plain structs standing in for geometry_msgs / lvr2 types (ROS 2 and lvr2 are not available in
// this image; the pluginlib shims that wrap these classes are sketched in INTEGRATION.md).
// All compute happens in libmeshnav_b200.so on the GPU.  Header-only; link with -lmeshnav_b200.
#pragma once
#include <array>
#include <cmath>
#include <cstdint>
#include <limits>
#include <list>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../meshnav_b200.h"

namespace meshnav_b200 {

struct Vector { float x = 0, y = 0, z = 0; };                       // mesh_map::Vector = lvr2::BaseVector<float>
inline Vector operator-(const Vector& a, const Vector& b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline float length(const Vector& v) { return std::sqrt(v.x * v.x + v.y * v.y + v.z * v.z); }
inline Vector normalized(const Vector& v) { const float l = length(v); return l > 0 ? Vector{v.x / l, v.y / l, v.z / l} : v; }

struct Quaternion { double x = 0, y = 0, z = 0, w = 1; };            // geometry_msgs::msg::Quaternion
struct PoseStamped {                                                // geometry_msgs::msg::PoseStamped (position + heading)
  Vector position;
  Vector direction;                                                 // unit vector along the path (orientation's x axis)
  Quaternion orientation;                                           // x axis along `direction`, z axis along the surface normal
};
inline Vector cross(const Vector& a, const Vector& b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

// mesh_map::calculatePoseFromDirection (mesh_map/src/util.cpp:267-287): basis ez = n, ey = n x dir, ex = ey x n (each
// normalised), columns of the rotation matrix; quaternion by tf2::Matrix3x3::getRotation (un-vendored ROS dependency,
// restated: trace / largest-diagonal branches) followed by normalize().
inline Quaternion calculatePoseFromDirection(const Vector& direction, const Vector& normal) {
  const Vector ez = normalized(normal), ey = normalized(cross(normal, direction)), ex = normalized(cross(ey, normal));
  const double m[3][3] = {{ex.x, ey.x, ez.x}, {ex.y, ey.y, ez.y}, {ex.z, ey.z, ez.z}};
  double t[4];
  const double trace = m[0][0] + m[1][1] + m[2][2];
  if (trace > 0.0) {
    double s = std::sqrt(trace + 1.0);
    t[3] = s * 0.5; s = 0.5 / s;
    t[0] = (m[2][1] - m[1][2]) * s; t[1] = (m[0][2] - m[2][0]) * s; t[2] = (m[1][0] - m[0][1]) * s;
  } else {
    const int i = m[0][0] < m[1][1] ? (m[1][1] < m[2][2] ? 2 : 1) : (m[0][0] < m[2][2] ? 2 : 0);
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    double s = std::sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0);
    t[i] = s * 0.5; s = 0.5 / s;
    t[3] = (m[k][j] - m[j][k]) * s; t[j] = (m[j][i] + m[i][j]) * s; t[k] = (m[k][i] + m[i][k]) * s;
  }
  const double l = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2] + t[3] * t[3]);
  return {t[0] / l, t[1] / l, t[2] / l, t[3] / l};
}

// outcome codes: mbf_msgs::action::GetPath::Result (dijkstra_mesh_planner.h:72-85)
enum : uint32_t { SUCCESS = 0, CANCELED = 51, INVALID_START = 52, INVALID_GOAL = 53, NO_PATH_FOUND = 54, INTERNAL_ERROR = 59 };

// The slice of mesh_map::MeshMap the hot path touches (mesh_map/include/mesh_map/mesh_map.h:97-452).
class MeshMap {
 public:
  MeshMap(const std::vector<float>& pos, const std::vector<uint32_t>& faces, int device = 0) : pos_(pos), faces_(faces) {
    if (mnb_create(device, &ctx_) != MNB_OK) throw std::runtime_error("meshnav_b200: no usable sm_90 device (no CPU fallback)");
    if (mnb_set_mesh(ctx_, (uint32_t)(pos.size() / 3), (uint32_t)(faces.size() / 3), pos.data(), faces.data(), nullptr, 0) != MNB_OK)
      throw std::runtime_error(mnb_last_error(ctx_));
    vertex_costs_.assign(numVertices(), 0.0f);
    edge_distances_.resize(numEdges());
    mnb_get_edge_distances(ctx_, edge_distances_.data());
    edge_weights_ = edge_distances_;
    invalid_.assign(numVertices(), 0);
  }
  ~MeshMap() { mnb_destroy(ctx_); }
  MeshMap(const MeshMap&) = delete;
  MeshMap& operator=(const MeshMap&) = delete;

  uint32_t numVertices() const { return mnb_num_vertices(ctx_); }
  uint32_t numFaces() const { return mnb_num_faces(ctx_); }
  uint32_t numEdges() const { return mnb_num_edges(ctx_); }
  mnb_ctx* ctx() const { return ctx_; }
  Vector vertexPosition(uint32_t v) const { return {pos_[3 * v], pos_[3 * v + 1], pos_[3 * v + 2]}; }
  const std::vector<uint32_t>& faces() const { return faces_; }
  // MeshMap::faceNormals()[f] (lvr2::calcFaceNormals, mesh_map.cpp:351): normalize(cross(p1 - p0, p2 - p0))
  Vector faceNormal(uint32_t f) const {
    const Vector p0 = vertexPosition(faces_[3 * (size_t)f]), p1 = vertexPosition(faces_[3 * (size_t)f + 1]), p2 = vertexPosition(faces_[3 * (size_t)f + 2]);
    return normalized(cross(p1 - p0, p2 - p0));
  }
  // MeshMap::vertexNormals()[v] (mesh_map.h:334; computed by mnb_set_mesh, fetched once)
  Vector vertexNormal(uint32_t v) const {
    if (vertex_normals_.empty()) { vertex_normals_.resize(3 * (size_t)numVertices()); mnb_get_vertex_normals(ctx_, vertex_normals_.data()); }
    return {vertex_normals_[3 * (size_t)v], vertex_normals_[3 * (size_t)v + 1], vertex_normals_[3 * (size_t)v + 2]};
  }
  std::vector<float>& vertexCosts() { return vertex_costs_; }          // MeshMap::vertexCosts()
  std::vector<float>& edgeWeights() { return edge_weights_; }          // MeshMap::edgeWeights()
  const std::vector<float>& edgeDistances() const { return edge_distances_; }
  std::vector<uint8_t>& invalid() { return invalid_; }                 // MeshMap::invalid (mesh_map.h:447)
  double edge_cost_factor = 0.0;                                       // mesh_map.cpp:105

  // MeshMap::computeEdgeWeights (mesh_map.cpp:517-561)
  bool computeEdgeWeights() {
    return mnb_compute_edge_weights(ctx_, vertex_costs_.data(), edge_cost_factor, edge_weights_.data()) == MNB_OK;
  }
  // pushes vertex_costs / edge_weights / invalid the way the planners read them (cvp:245,663-664)
  bool syncCosts() { return mnb_set_costs(ctx_, vertex_costs_.data(), edge_weights_.data(), invalid_.data()) == MNB_OK; }

  // MeshMap::layerChanged (mesh_map.cpp:455-492): vertex_costs of the changed vertices from the default layer's cost map
  // (NaN = no entry -> default_value), then updateEdgeWeights (:563-618) -- on the device only the table entries of the
  // incident edges are patched; the host copies are refreshed from the device.
  bool layerChanged(const std::vector<uint32_t>& changes, const std::vector<float>& layer_costs, float default_value) {
    if (layer_costs.size() != vertex_costs_.size()) return false;
    if (mnb_update_vertex_costs(ctx_, (uint32_t)changes.size(), changes.data(), layer_costs.data(), 1, default_value, edge_cost_factor) != MNB_OK)
      return false;
    return mnb_get_costs(ctx_, vertex_costs_.data(), edge_weights_.data()) == MNB_OK;
  }

  // MeshMap::getNearestVertexHandle (mesh_map.cpp:1161-1174): one streamed pass over the device-resident positions
  int64_t getNearestVertexHandle(const Vector& p) const {
    uint32_t v = 0;
    return mnb_locate(ctx_, 1, &p.x, &v, nullptr, nullptr) == MNB_OK ? (int64_t)v : -1;
  }
  // MeshMap::getContainingFace / searchContainingFace (mesh_map.cpp:1110-1159); like the reference, max_dist is
  // accepted but not consulted.  -1 = no containing face.
  int64_t getContainingFace(const Vector& p, float /*max_dist*/) const {
    int32_t f = -1;
    return mnb_locate(ctx_, 1, &p.x, nullptr, &f, nullptr) == MNB_OK ? (int64_t)f : -1;
  }
  // MeshMap::searchContainingFace (mesh_map.cpp:1120-1159) with the barycentric coordinates
  bool searchContainingFace(const Vector& p, uint32_t& face, float bary[3]) const {
    int32_t f = -1;
    if (mnb_locate(ctx_, 1, &p.x, nullptr, &f, bary) != MNB_OK || f < 0) return false;
    face = (uint32_t)f;
    return true;
  }

 private:
  mnb_ctx* ctx_ = nullptr;
  std::vector<float> pos_; std::vector<uint32_t> faces_;
  std::vector<float> vertex_costs_, edge_weights_, edge_distances_;
  mutable std::vector<float> vertex_normals_;
  std::vector<uint8_t> invalid_;
};

// mbf_mesh_core::MeshPlanner (mesh_planner.h:50-92)
class MeshPlanner {
 public:
  virtual ~MeshPlanner() = default;
  virtual uint32_t makePlan(const PoseStamped& start, const PoseStamped& goal, double tolerance,
                            std::vector<PoseStamped>& plan, double& cost, std::string& message) = 0;     // :71-73
  virtual bool cancel() = 0;                                                                                // :80
  virtual bool initialize(const std::string& name, const std::shared_ptr<MeshMap>& mesh_map_ptr) = 0;       // :88
};

class DijkstraMeshPlanner : public MeshPlanner {
 public:
  struct { double goal_dist_offset = 0.3; double cost_limit = 1.0; } config_;     // dijkstra_mesh_planner.h:178-187

  bool initialize(const std::string& name, const std::shared_ptr<MeshMap>& mesh_map_ptr) override {
    name_ = name; mesh_map_ = mesh_map_ptr; return true;
  }
  bool cancel() override { return mnb_cancel(mesh_map_->ctx()) == MNB_OK; }                   // dijkstra_mesh_planner.cpp:136-140

  // dijkstra_mesh_planner.cpp:55-134: the wave is seeded at the GOAL, the robot (start) is the target
  uint32_t makePlan(const PoseStamped& start, const PoseStamped& goal, double /*tolerance*/, std::vector<PoseStamped>& plan,
                    double& cost, std::string& message) override {
    std::list<uint32_t> path;
    const uint32_t outcome = dijkstra(goal.position, start.position, path);     // :81
    path.reverse();                                                              // :83
    cost = 0;
    if (!path.empty()) {                                                         // :90-116
      Vector vec = start.position;
      Vector normal = mesh_map_->vertexNormal(path.front());                     // :93-94
      while (!path.empty()) {
        const uint32_t vH = path.front();
        const Vector next = mesh_map_->vertexPosition(vH);
        PoseStamped pose; pose.position = vec; pose.direction = normalized(next - vec);
        pose.orientation = calculatePoseFromDirection(next - vec, normal);       // :106 calculatePoseFromPosition(vec, next, normal)
        cost += length(next - vec);
        vec = next;
        normal = mesh_map_->vertexNormal(vH);                                    // :109
        plan.push_back(pose);
        path.pop_front();
      }
      PoseStamped pose; pose.position = vec; pose.direction = normalized(goal.position - vec);
      pose.orientation = calculatePoseFromDirection(goal.position - vec, normal);   // :113
      cost += length(goal.position - vec);
      plan.push_back(pose);
    }
    if (outcome == NO_PATH_FOUND) message = "Predecessor of the goal is not set! No path found!";
    return outcome;
  }

  // dijkstra_mesh_planner.cpp:211-398 (original_start = wave seed, original_goal = robot)
  uint32_t dijkstra(const Vector& original_start, const Vector& original_goal, std::list<uint32_t>& path) {
    const int64_t start_vertex = mesh_map_->getNearestVertexHandle(original_start);   // :235
    const int64_t goal_vertex = mesh_map_->getNearestVertexHandle(original_goal);     // :236
    if (start_vertex < 0) return INVALID_START;
    if (goal_vertex < 0) return INVALID_GOAL;
    path.clear();
    if (goal_vertex == start_vertex) return SUCCESS;                                   // :252-255
    const uint32_t V = mesh_map_->numVertices();
    potential_.assign(V, 0.0f); predecessors_.assign(V, 0);
    if (!mesh_map_->syncCosts()) return INTERNAL_ERROR;
    const int32_t rc = mnb_dijkstra(mesh_map_->ctx(), (uint32_t)start_vertex, goal_vertex, config_.cost_limit,
                                    config_.goal_dist_offset, potential_.data(), predecessors_.data());
    if (rc < 0) return INTERNAL_ERROR;
    if (rc != SUCCESS) return (uint32_t)rc;
    uint32_t vH = (uint32_t)goal_vertex;                                               // :367-373
    while (vH != (uint32_t)start_vertex) { vH = predecessors_[vH]; path.push_front(vH); }
    computeVectorMap();                                                                // :380
    return SUCCESS;
  }

  // dijkstra_mesh_planner.cpp:189-209 (GPU epilogue; NaN row = no entry in the sparse map)
  void computeVectorMap() {
    vector_map_.assign(mesh_map_->numVertices(), Vector{});
    mnb_vector_map(mesh_map_->ctx(), predecessors_.data(), nullptr, nullptr, &vector_map_[0].x);
  }
  const std::vector<float>& potential() const { return potential_; }
  const std::vector<uint32_t>& predecessors() const { return predecessors_; }
  const std::vector<Vector>& getVectorMap() const { return vector_map_; }              // :171-174

 private:
  std::string name_; std::shared_ptr<MeshMap> mesh_map_;
  std::vector<float> potential_; std::vector<uint32_t> predecessors_; std::vector<Vector> vector_map_;
};

class CVPMeshPlanner : public MeshPlanner {
 public:
  struct { double goal_dist_offset = 0.3; double cost_limit = 1.0; double step_width = 0.4; } config_;   // cvp_mesh_planner.h:201-212

  bool initialize(const std::string& name, const std::shared_ptr<MeshMap>& mesh_map_ptr) override {
    name_ = name; mesh_map_ = mesh_map_ptr; return true;
  }
  bool cancel() override { return mnb_cancel(mesh_map_->ctx()) == MNB_OK; }                               // cvp:142-146

  // cvp_mesh_planner.cpp:62-140: wavefront seeded at the goal, then the vector-field back-tracking of :920-951
  // (MeshMap::meshAhead) on the device; `path` comes back in plan order (robot first), so the reference's
  // path.reverse() (:100) is already applied.  Poses: position + direction to the next point (:104-120).
  uint32_t makePlan(const PoseStamped& start, const PoseStamped& goal, double /*tolerance*/, std::vector<PoseStamped>& plan,
                    double& cost, std::string& message) override {
    std::vector<std::pair<Vector, uint32_t>> path;
    const uint32_t outcome = waveFrontPropagation(goal.position, start.position, path, message);         // :89
    cost = 0;
    if (!path.empty()) {
      Vector vec = path.front().first;                                                                    // :104-120
      for (size_t i = 1; i < path.size(); ++i) {
        const Vector next = path[i].first;
        PoseStamped pose; pose.position = vec; pose.direction = normalized(next - vec);
        pose.orientation = calculatePoseFromDirection(next - vec, mesh_map_->faceNormal(path[i - 1].second));   // :112 calculatePoseFromPosition
        cost += length(next - vec);
        vec = next;
        plan.push_back(pose);
      }
      PoseStamped pose = goal; pose.position = vec;                                                       // :121-125 goal pose, caller's orientation
      if (!plan.empty() && length(goal.direction) == 0.0f) pose.direction = plan.back().direction;
      plan.push_back(pose);
    }
    return outcome;
  }

  // cvp_mesh_planner.cpp:651-970 including the back-tracking; path in plan order (robot ... wave seed)
  uint32_t waveFrontPropagation(const Vector& start, const Vector& goal, std::vector<std::pair<Vector, uint32_t>>& path,
                                std::string& message) {
    path.clear();
    const uint32_t outcome = waveFrontPropagation(start, goal, message);
    if (outcome != SUCCESS) return outcome;
    computeVectorMap();                                                                                   // :897
    const int64_t goal_face = mesh_map_->getContainingFace(goal, 0.4f);
    const uint32_t max_points = 1u << 16;
    std::vector<float> pp(3 * (size_t)max_points); std::vector<uint32_t> pf(max_points);
    uint32_t n = 0;
    const float gp[3] = {goal.x, goal.y, goal.z};
    const int32_t rc = mnb_cvp_backtrack(mesh_map_->ctx(), gp, (uint32_t)goal_face, config_.step_width, max_points, pp.data(),
                                         pf.data(), &n);
    if (rc < 0) { message = mnb_last_error(mesh_map_->ctx()); return INTERNAL_ERROR; }
    if (rc == NO_PATH_FOUND) { message = "Could not find a valid path, while back-tracking from the goal"; return NO_PATH_FOUND; }   // :938-941
    if (rc != SUCCESS) return (uint32_t)rc;
    for (uint32_t i = 0; i < n; ++i) path.push_back({Vector{pp[3 * i], pp[3 * i + 1], pp[3 * i + 2]}, pf[i]});
    return SUCCESS;
  }

  // cvp_mesh_planner.cpp:204-239 (GPU epilogue; NaN row = no entry in the sparse map)
  void computeVectorMap() {
    vector_map_.assign(mesh_map_->numVertices(), Vector{});
    mnb_vector_map(mesh_map_->ctx(), predecessors_.data(), direction_.data(), cutting_faces_.data(), &vector_map_[0].x);
  }
  const std::vector<Vector>& getVectorMap() const { return vector_map_; }                                // :200-203

  // cvp_mesh_planner.cpp:241-247, 651-970 (propagation part)
  uint32_t waveFrontPropagation(const Vector& start, const Vector& goal, std::string& message) {
    const int64_t start_face = mesh_map_->getContainingFace(start, 0.4f);                                // :673
    const int64_t goal_face = mesh_map_->getContainingFace(goal, 0.4f);                                  // :674
    if (start_face < 0) { message = "Could not find a face close enough to the given start pose"; return INVALID_START; }   // :681-685
    if (goal_face < 0) { message = "Could not find a face close enough to the given goal pose"; return INVALID_GOAL; }     // :686-690
    const uint32_t V = mesh_map_->numVertices();
    potential_.assign(V, 0.0f); predecessors_.assign(V, 0); direction_.assign(V, 0.0f); cutting_faces_.assign(V, -1);
    if (!mesh_map_->syncCosts()) return INTERNAL_ERROR;
    const float sp[3] = {start.x, start.y, start.z};
    const int32_t rc = mnb_cvp(mesh_map_->ctx(), (uint32_t)start_face, sp, goal_face, config_.cost_limit, config_.goal_dist_offset,
                               potential_.data(), predecessors_.data(), direction_.data(), cutting_faces_.data());
    if (rc < 0) { message = mnb_last_error(mesh_map_->ctx()); return INTERNAL_ERROR; }
    if (rc == NO_PATH_FOUND) message = "Predecessor of the goal is not set! No path found!";             // :915
    return (uint32_t)rc;
  }
  const std::vector<float>& potential() const { return potential_; }
  const std::vector<uint32_t>& predecessors() const { return predecessors_; }
  const std::vector<float>& direction() const { return direction_; }
  const std::vector<int32_t>& cuttingFaces() const { return cutting_faces_; }

 private:
  std::string name_; std::shared_ptr<MeshMap> mesh_map_;
  std::vector<float> potential_, direction_; std::vector<uint32_t> predecessors_; std::vector<int32_t> cutting_faces_;
  std::vector<Vector> vector_map_;
};

// mesh_layers::InflationLayer -- waveCostInflation + fading (inflation_layer.cpp:315-491)
class InflationLayer {
 public:
  struct {                                                           // inflation_layer.h:240-248
    double inscribed_radius = 0.25, inflation_radius = 0.4, lethal_value = 1.0, inscribed_value = 0.99,
           cost_scaling_factor = 1.0;
  } config_;
  explicit InflationLayer(const std::shared_ptr<MeshMap>& map) : map_(map) {}

  // returns false on error; riskiness (NaN = not in the sparse map) and distances (+inf = not in the map)
  bool waveCostInflation(const std::vector<uint32_t>& lethals, std::vector<float>& cost_out, std::vector<float>& distances) {
    const uint32_t V = map_->numVertices();
    cost_out.assign(V, 0.0f); distances.assign(V, 0.0f);
    const mnb_inflation_params p{config_.inscribed_radius, config_.inflation_radius, config_.lethal_value,
                                 config_.inscribed_value, config_.cost_scaling_factor};
    return mnb_inflate(map_->ctx(), lethals.data(), (uint32_t)lethals.size(), map_->invalid().data(), &p, distances.data(),
                       cost_out.data()) == MNB_OK;
  }

  // InflationLayer::onInputChanged (inflation_layer.cpp:97-179): full re-inflation from the input layer's lethals; `update`
  // receives the set handed to notifyChange (:154-176).  riskiness_ / distances_ are kept as members like in the reference.
  bool onInputChanged(const std::vector<uint32_t>& lethals, std::vector<uint32_t>& update) {
    const uint32_t V = map_->numVertices();
    riskiness_.assign(V, 0.0f); distances_.assign(V, 0.0f); update.assign(V, 0u);
    const mnb_inflation_params p{config_.inscribed_radius, config_.inflation_radius, config_.lethal_value,
                                 config_.inscribed_value, config_.cost_scaling_factor};
    uint32_t n = 0;
    if (mnb_inflation_update(map_->ctx(), lethals.data(), (uint32_t)lethals.size(), map_->invalid().data(), &p, distances_.data(),
                             riskiness_.data(), update.data(), &n) != MNB_OK) return false;
    update.resize(n);
    return true;
  }
  const std::vector<float>& costs() const { return riskiness_; }      // AbstractLayer::costs(): NaN = no entry
  float defaultValue() const { return 0; }                            // inflation_layer.h:74-77

  // vector_map_ of the last wave (inflation_layer.cpp:277-308); call before the next plan on the same map
  bool vectorMap(std::vector<Vector>& out) {
    std::vector<float> raw(3 * (size_t)map_->numVertices());
    if (mnb_inflation_vector_map(map_->ctx(), raw.data()) != MNB_OK) return false;
    out.resize(map_->numVertices());
    for (size_t v = 0; v < out.size(); ++v) out[v] = {raw[3 * v], raw[3 * v + 1], raw[3 * v + 2]};
    return true;
  }
  // InflationLayer::vectorAt(vertices, barycentric_coords) (inflation_layer.cpp:493-521)
  Vector vectorAt(uint32_t face, const std::array<float, 3>& barycentric_coords) {
    Vector v;
    mnb_inflation_vector_at(map_->ctx(), 1, &face, barycentric_coords.data(), &v.x);
    return v;
  }

 private:
  std::shared_ptr<MeshMap> map_;
  std::vector<float> riskiness_, distances_;
};

// mesh_layers::ObstacleLayer (mesh_layers/src/obstacle_layer.cpp) without the ROS plumbing: the lethal set of the latest
// point cloud; costs: +inf on lethal vertices, no entry (NaN) elsewhere, defaultValue() 0, threshold() +inf.
class ObstacleLayer {
 public:
  struct {                                                           // obstacle_layer.h:142-151
    double robot_height = std::numeric_limits<double>::infinity();
    double max_obstacle_dist = std::numeric_limits<double>::infinity();
    Vector down_axis{0.0f, 0.0f, -1.0f};                             // normalised at configuration time (obstacle_layer.cpp:110)
  } config_;
  explicit ObstacleLayer(const std::shared_ptr<MeshMap>& map) : map_(map) { mnb_obstacle_reset(map_->ctx()); }

  // ObstacleLayer::processPointCloud (obstacle_layer.cpp:133-296): `points` in the message frame, `tf` the row-major 3x4
  // [R|t] into the map frame (:176-180), `axis_in_map` the down axis rotated into the map frame (:183-205).  `changed`
  // receives what notifyChange is called with (:268-296).
  bool processPointCloud(const std::vector<float>& points, const std::array<float, 12>& tf, const Vector& axis_in_map,
                         std::vector<uint32_t>& changed) {
    mnb_obstacle_params p{};
    p.max_obstacle_dist = config_.max_obstacle_dist; p.robot_height = config_.robot_height;
    for (int k = 0; k < 12; ++k) p.tf[k] = tf[k];
    p.down_axis[0] = axis_in_map.x; p.down_axis[1] = axis_in_map.y; p.down_axis[2] = axis_in_map.z;
    const uint32_t V = map_->numVertices();
    lethals_.assign(V, 0u); changed.assign(V, 0u); costs_.assign(V, 0.0f);
    uint32_t nl = 0, nc = 0;
    if (mnb_obstacle_update(map_->ctx(), (uint32_t)(points.size() / 3), points.data(), &p, lethals_.data(), &nl, changed.data(), &nc,
                            costs_.data()) != MNB_OK) return false;
    lethals_.resize(nl); changed.resize(nc);
    return true;
  }
  const std::vector<uint32_t>& lethals() const { return lethals_; }   // ascending (std::set order)
  const std::vector<float>& costs() const { return costs_; }          // NaN = no entry
  float defaultValue() const { return 0.0f; }                         // obstacle_layer.h:80
  float threshold() const { return std::numeric_limits<float>::infinity(); }   // :89

 private:
  std::shared_ptr<MeshMap> map_;
  std::vector<uint32_t> lethals_;
  std::vector<float> costs_;
};

// MeshMap::raycaster()->castRays (mesh_map.h:318, obstacle_layer.cpp:239) and lvr2::calcNormalClearance
// (clearance_layer.cpp:161) on the device BVH
struct RayCastResult { std::vector<uint8_t> hit; std::vector<float> dist; std::vector<uint32_t> face; std::vector<float> point; };
inline bool castRays(MeshMap& map, const std::vector<float>& origins, const std::vector<float>& dirs, RayCastResult& out) {
  const uint32_t n = (uint32_t)(origins.size() / 3);
  if (dirs.size() != 3 && dirs.size() != origins.size()) return false;
  out.hit.assign(n, 0); out.dist.assign(n, 0.0f); out.face.assign(n, 0u); out.point.assign(3 * (size_t)n, 0.0f);
  return mnb_cast_rays(map.ctx(), n, origins.data(), dirs.data(), dirs.size() == 3 && n != 1 ? 0u : 3u, out.hit.data(), out.dist.data(),
                       out.face.data(), out.point.data()) == MNB_OK;
}
inline bool calcNormalClearance(MeshMap& map, std::vector<float>& clearance) {
  clearance.assign(map.numVertices(), 0.0f);
  return mnb_normal_clearance(map.ctx(), nullptr, clearance.data()) == MNB_OK;
}

}  // namespace meshnav_b200
