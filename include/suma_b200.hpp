// suma_b200.hpp -- header-only C++ mirror of the reference's boundary classes on top of the C ABI (suma_b200.h).
//
// Same class names, method names and argument meaning as PRBonn/semantic_suma's core/ headers, so that code written
// against SurfelMapping / Frame2Model / LieGaussNewton / SurfelMap / Preprocessing / Frame keeps compiling:
//   core/SurfelMapping.h:33-109, core/Frame2Model.h:28-73, core/Objective.h:14-82, core/LieGaussNewton.h:25-77,
//   core/SurfelMap.h:36-78, core/Preprocessing.h:47-58, core/Frame.h:21-79.
// Differences that a maintainer has to know (INTEGRATION.md):
//   * matrices are suma::Matrix4f / Matrix4d (16 column-major values). With -DSUMA_B200_WITH_EIGEN they convert
//     from/to Eigen::Matrix4f / Matrix4d implicitly.
//   * rv::ParameterList -> suma::ParameterList (string-keyed, same XML key names); rv::Laserscan -> suma::Laserscan.
//   * the GL objects inside Frame (GlTextureRectangle) become device images; use Frame::download*() or the optional
//     CUDA-GL interop described in INTEGRATION.md for display.
//   * errors: the reference throws std::runtime_error; so does this shim (from negative sb_status codes).
#ifndef SUMA_B200_HPP_
#define SUMA_B200_HPP_

#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "suma_b200.h"

#ifdef SUMA_B200_WITH_EIGEN
#include <Eigen/Dense>
#endif

namespace suma {

template <typename T>
struct Matrix4 {
  T m[16];  // column-major, like Eigen
  Matrix4() { setIdentity(); }
  void setIdentity() {
    for (int i = 0; i < 16; ++i) m[i] = (i % 5 == 0) ? T(1) : T(0);
  }
  static Matrix4 Identity() { return Matrix4(); }
  T& operator()(int r, int c) { return m[c * 4 + r]; }
  const T& operator()(int r, int c) const { return m[c * 4 + r]; }
  T* data() { return m; }
  const T* data() const { return m; }
  template <typename U>
  Matrix4<U> cast() const {
    Matrix4<U> r;
    for (int i = 0; i < 16; ++i) r.m[i] = static_cast<U>(m[i]);
    return r;
  }
  Matrix4 operator*(const Matrix4& B) const {  // same evaluation order as the library (sb_math.cuh mat4_mul)
    Matrix4 C;
    for (int c = 0; c < 4; ++c)
      for (int r = 0; r < 4; ++r)
        C.m[c * 4 + r] = ((m[0 * 4 + r] * B.m[c * 4 + 0] + m[1 * 4 + r] * B.m[c * 4 + 1]) + m[2 * 4 + r] * B.m[c * 4 + 2]) +
                         m[3 * 4 + r] * B.m[c * 4 + 3];
    return C;
  }
#ifdef SUMA_B200_WITH_EIGEN
  Matrix4(const Eigen::Matrix<T, 4, 4>& e) { std::memcpy(m, e.data(), sizeof(m)); }
  operator Eigen::Matrix<T, 4, 4>() const {
    Eigen::Matrix<T, 4, 4> e;
    std::memcpy(e.data(), m, sizeof(m));
    return e;
  }
#endif
};
using Matrix4f = Matrix4<float>;
using Matrix4d = Matrix4<double>;

struct Vector6d {
  double v[6];
  double& operator[](int i) { return v[i]; }
  const double& operator[](int i) const { return v[i]; }
};
struct Matrix6d {
  double m[36];  // column-major
  double& operator()(int r, int c) { return m[c * 6 + r]; }
};

/** stand-in for rv::ParameterList: string keys as in config/default.xml */
class ParameterList {
 public:
  ParameterList() { sb_default_params(&p_); }
  explicit ParameterList(const sb_params& p) : p_(p) {}
  bool hasParam(const std::string& k) const { return fields().count(k) > 0; }
  void insert(const std::string& key, double value) {
    if (key == "weighting") {
      p_.weighting = static_cast<int32_t>(value);
      return;
    }
    auto it = fields().find(key);
    if (it == fields().end()) throw std::runtime_error("suma::ParameterList: unknown parameter " + key);
    const Field& f = it->second;
    char* base = reinterpret_cast<char*>(&p_);
    if (f.kind == 0) *reinterpret_cast<int32_t*>(base + f.off) = static_cast<int32_t>(value);
    if (f.kind == 1) *reinterpret_cast<float*>(base + f.off) = static_cast<float>(value);
    if (f.kind == 2) *reinterpret_cast<double*>(base + f.off) = value;
  }
  void insert(const std::string& key, const std::string& value) {  // "weighting" = none|huber|turkey|stability
    if (key != "weighting") throw std::runtime_error("suma::ParameterList: string parameter " + key);
    p_.weighting = value == "huber" ? 1 : value == "turkey" ? 2 : value == "stability" ? 3 : 0;
  }
  const sb_params& raw() const { return p_; }
  sb_params& raw() { return p_; }

 private:
  struct Field {
    size_t off;
    int kind;
  };
#define SUMA_F(name, member, kind) {name, Field{offsetof(sb_params, member), kind}}
  static const std::map<std::string, Field>& fields() {
    static const std::map<std::string, Field> f = {
        SUMA_F("data_width", data_width, 0), SUMA_F("data_height", data_height, 0),
        SUMA_F("data_fov_up", data_fov_up, 1), SUMA_F("data_fov_down", data_fov_down, 1),
        SUMA_F("min_depth", min_depth, 1), SUMA_F("max_depth", max_depth, 1),
        SUMA_F("model_width", model_width, 0), SUMA_F("model_height", model_height, 0),
        SUMA_F("model_fov_up", model_fov_up, 1), SUMA_F("model_fov_down", model_fov_down, 1),
        SUMA_F("model_min_depth", model_min_depth, 1), SUMA_F("model_max_depth", model_max_depth, 1),
        SUMA_F("max iterations", max_iterations, 0), SUMA_F("stopping threshold", stopping_threshold, 2),
        SUMA_F("delta", delta, 2), SUMA_F("icp-max-distance", icp_max_distance, 1),
        SUMA_F("icp-max-angle", icp_max_angle, 1), SUMA_F("factor", factor, 1),
        SUMA_F("initialize_identity", initialize_identity, 0), SUMA_F("bilinear_sampling", bilinear_sampling, 0),
        SUMA_F("fallback_mode", fallback_mode, 0), SUMA_F("fallback-max-distance", fallback_max_distance, 1),
        SUMA_F("fallback-max-angle", fallback_max_angle, 1), SUMA_F("compose_rendering", compose_rendering, 0),
        SUMA_F("max_loop_closure_distance", max_loop_closure_distance, 1), SUMA_F("min_radius", min_radius, 1),
        SUMA_F("max_radius", max_radius, 1), SUMA_F("max_angle", max_angle, 1),
        SUMA_F("map-max-distance", map_max_distance, 1), SUMA_F("map-max-angle", map_max_angle, 1),
        SUMA_F("unstable_age", unstable_age, 0), SUMA_F("confidence_mode", confidence_mode, 0),
        SUMA_F("confidence_threshold", confidence_threshold, 1), SUMA_F("p_stable", p_stable, 1),
        SUMA_F("p_prior", p_prior, 1), SUMA_F("sigma_angle", sigma_angle, 1),
        SUMA_F("sigma_distance", sigma_distance, 1), SUMA_F("use_stability", use_stability, 0),
        SUMA_F("active_timestamps", active_timestamps, 0), SUMA_F("max_weight", max_weight, 1),
        SUMA_F("weighting_scheme", weighting_scheme, 0), SUMA_F("averaging_scheme", averaging_scheme, 0),
        SUMA_F("update_always", update_always, 0), SUMA_F("submap-dimension", submap_dimension, 0),
        SUMA_F("submap-extent", submap_extent, 1), SUMA_F("partial-extraction", partial_extraction, 0),
        SUMA_F("label_offset_quirk", label_offset_quirk, 0), SUMA_F("render_after_update", render_after_update, 0),
    };
    return f;
  }
#undef SUMA_F
  sb_params p_;
};

/** stand-in for rv::Laserscan (io/KITTIReader.cpp:136-203 fills points, labels_float, labels_prob) */
struct Laserscan {
  std::vector<float> points;  // x, y, z, 1 per point (rv::Point3f = Eigen::Vector4f, rv/geometry.h:331-345)
  std::vector<float> labels_float;
  std::vector<float> labels_prob;
  uint32_t size() const { return static_cast<uint32_t>(points.size() / 4); }
};

inline void check(int rc, sb_ctx* ctx, const char* what) {
  if (rc != SB_OK) throw std::runtime_error(std::string(what) + ": " + (ctx ? sb_last_error(ctx) : "") + " (status " + std::to_string(rc) + ")");
}

/** one CUDA device + stream: the role the Qt-owned GL context plays in the reference */
class Context {
 public:
  explicit Context(const ParameterList& params, int device = 0) : params_(params) {
    int rc = sb_create(&params_.raw(), device, &ctx_);
    if (rc != SB_OK) throw std::runtime_error("sb_create failed with status " + std::to_string(rc) + " (libsuma_b200 needs a CUDA device)");
  }
  ~Context() {
    if (ctx_) sb_destroy(ctx_);
  }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  sb_ctx* get() const { return ctx_; }
  const ParameterList& params() const { return params_; }
  void setParameters(const ParameterList& p) {
    check(sb_set_params(ctx_, &p.raw()), ctx_, "setParameters");
    params_ = p;
  }
  /** the parameters the library already holds (after sb_state_load) */
  void adoptParameters(const ParameterList& p) { params_ = p; }

 private:
  ParameterList params_;
  sb_ctx* ctx_{nullptr};
};
using ContextPtr = std::shared_ptr<Context>;

/** core/Frame.h */
class Frame {
 public:
  typedef std::shared_ptr<Frame> Ptr;
  Frame(const ContextPtr& ctx, uint32_t w, uint32_t h) : width(w), height(h), ctx_(ctx), owned_(true) {
    check(sb_frame_create(ctx->get(), static_cast<int>(w), static_cast<int>(h), &f_), ctx->get(), "Frame");
  }
  Frame(const ContextPtr& ctx, sb_frame* borrowed) : ctx_(ctx), f_(borrowed), owned_(false) {  // not owned
    int w = 0, h = 0;
    sb_frame_size(f_, &w, &h);
    width = static_cast<uint32_t>(w);
    height = static_cast<uint32_t>(h);
  }
  ~Frame() {
    if (owned_ && f_) sb_frame_destroy(f_);
  }
  Frame(const Frame&) = delete;
  void copy(const Frame& other) { check(sb_frame_copy(f_, other.f_), ctx_->get(), "Frame::copy"); }
  std::vector<float> download(int which) const {
    std::vector<float> a(static_cast<size_t>(width) * height * 4);
    check(sb_frame_download(f_, which, a.data()), ctx_->get(), "Frame::download");
    return a;
  }
  std::vector<float> vertex_map() const { return download(SB_MAP_VERTEX); }
  std::vector<float> normal_map() const { return download(SB_MAP_NORMAL); }
  std::vector<float> semantic_map() const { return download(SB_MAP_SEMANTIC); }
  sb_frame* handle() const { return f_; }
  bool valid{false};
  uint32_t width{0}, height{0};
  Matrix4f pose;

 private:
  ContextPtr ctx_;
  sb_frame* f_{nullptr};
  bool owned_;
};

/** core/Preprocessing.h */
class Preprocessing {
 public:
  explicit Preprocessing(const ContextPtr& ctx) : ctx_(ctx) {}
  void setParameters(const ParameterList& params) { ctx_->setParameters(params); }
  /** Preprocessing.cpp:341 stores the calibration "for semantic map"; no pass of the hot path reads it */
  template <class Calibration>
  void setCalibration(const Calibration&) {}
  /** Preprocessing::process(points, frame, labels, probs, timestamp), Preprocessing.cpp:120 */
  void process(const std::vector<float>& points, Frame& frame, const std::vector<float>& labels,
               const std::vector<float>& probs, uint32_t timestamp) {
    uint32_t n = static_cast<uint32_t>(points.size() / 4);
    check(sb_preprocess(ctx_->get(), points.data(), labels.empty() ? nullptr : labels.data(),
                        probs.empty() ? nullptr : probs.data(), n, timestamp, 0, frame.handle()),
          ctx_->get(), "Preprocessing::process");
    frame.valid = true;
  }

 private:
  ContextPtr ctx_;
};

/** core/Objective.h + core/Frame2Model.h */
class Objective {
 public:
  virtual ~Objective() {}
  virtual uint32_t num_parameters() const = 0;
  virtual void setData(const std::shared_ptr<Frame>& current, const std::shared_ptr<Frame>& last) = 0;
  virtual double jacobianProducts(Matrix6d& JtJ, Vector6d& Jtf) = 0;
  void increment(const Vector6d& delta) {
    Matrix4d E;
    sb_se3_exp(delta.v, E.m);
    pose_ = E * pose_;
    iteration_ += 1;
  }
  uint32_t inlier() const { return inlier_; }
  uint32_t outlier() const { return outlier_; }
  uint32_t valid() const { return inlier_ + outlier_; }
  uint32_t invalid() const { return invalid_; }
  float inlier_residual() const { return inlier_residual_; }
  void initialize(const Matrix4d& T0) { pose_ = T0; }
  const Matrix4d& pose() const { return pose_; }

 protected:
  Matrix4d pose_;
  uint32_t iteration_{0}, inlier_{0}, outlier_{0}, invalid_{0};
  float inlier_residual_{0.0f};
};

class Frame2Model : public Objective {
 public:
  explicit Frame2Model(const ContextPtr& ctx) : ctx_(ctx) {
    max_distance_ = ctx->params().raw().icp_max_distance;
    max_angle_ = ctx->params().raw().icp_max_angle;
  }
  Frame2Model(const ContextPtr& ctx, float max_distance, float max_angle)
      : ctx_(ctx), max_distance_(max_distance), max_angle_(max_angle) {}
  void setData(const std::shared_ptr<Frame>& current, const std::shared_ptr<Frame>& last) override {
    current_ = current;
    last_ = last;
    iteration_ = 0;
  }
  uint32_t num_parameters() const override { return 6; }
  double jacobianProducts(Matrix6d& JtJ, Vector6d& Jtf) override {
    double o[48];
    check(sb_icp_jacobian(ctx_->get(), current_->handle(), last_->handle(), pose_.m, static_cast<int>(iteration_),
                          max_distance_, max_angle_, 0, static_cast<int>(current_->height), o, nullptr),
          ctx_->get(), "Frame2Model::jacobianProducts");
    std::memcpy(JtJ.m, o, sizeof(JtJ.m));
    std::memcpy(Jtf.v, o + 36, sizeof(Jtf.v));
    uint32_t valid = static_cast<uint32_t>(o[42]);  // Frame2Model.cpp:222-227
    outlier_ = static_cast<uint32_t>(o[44]);
    inlier_residual_ = static_cast<float>(o[45]);
    inlier_ = valid - outlier_;
    invalid_ = static_cast<uint32_t>(o[46]);
    return o[43];
  }
  const std::shared_ptr<Frame>& current() const { return current_; }
  const std::shared_ptr<Frame>& last() const { return last_; }
  float max_distance() const { return max_distance_; }
  float max_angle() const { return max_angle_; }
  void absorb(const double pose[16], const double o[48], int iterations) {  // result of the fused device loop
    std::memcpy(pose_.m, pose, sizeof(pose_.m));
    iteration_ = static_cast<uint32_t>(iterations);
    outlier_ = static_cast<uint32_t>(o[44]);
    inlier_ = static_cast<uint32_t>(o[42]) - outlier_;
    invalid_ = static_cast<uint32_t>(o[46]);
    inlier_residual_ = static_cast<float>(o[45]);
  }

 private:
  ContextPtr ctx_;
  std::shared_ptr<Frame> current_, last_;
  float max_distance_, max_angle_;
};

/** core/LieGaussNewton.h */
class LieGaussNewton {
 public:
  explicit LieGaussNewton(const ContextPtr& ctx) : ctx_(ctx) { setParameters(ctx->params()); }
  void setParameters(const ParameterList& params) {
    maxIter = static_cast<uint32_t>(params.raw().max_iterations);
    epsilon = params.raw().stopping_threshold;
    delta = params.raw().delta;
  }
  /** minimize(F, T0): the whole loop runs on the device when F is a Frame2Model (no host round trip per iteration) */
  int32_t minimize(Objective& F, const Matrix4d& T0) {
    history_.clear();
    if (Frame2Model* f2m = dynamic_cast<Frame2Model*>(&F)) {
      double pose[16], o[48];
      int iters = 0, hl = 0;
      std::vector<double> hist(static_cast<size_t>(maxIter > 0 ? maxIter + 2 : 258) * 16);
      check(sb_icp_minimize(ctx_->get(), f2m->current()->handle(), f2m->last()->handle(), T0.m, static_cast<int>(maxIter),
                            epsilon, delta, f2m->max_distance(), f2m->max_angle(), pose, o, &iters, hist.data(), &hl),
            ctx_->get(), "LieGaussNewton::minimize");
      f2m->absorb(pose, o, iters);
      std::memcpy(Tk_.m, pose, sizeof(Tk_.m));
      k_ = static_cast<uint32_t>(iters);
      last_error = o[43];
      for (int i = 0; i < hl; ++i) {
        Matrix4d h;
        std::memcpy(h.m, hist.data() + 16 * i, sizeof(h.m));
        history_.push_back(h);
      }
      return 0;
    }
    // generic objective: the reference's host loop (LieGaussNewton.cpp:13-37) with the library's solver
    F.initialize(T0);
    Tk_ = T0;
    last_error = 3.402823466e+38;
    k_ = 0;
    for (;;) {
      history_.push_back(Tk_);
      if (maxIter > 0 && k_ >= maxIter) break;
      Matrix6d JtJ;
      Vector6d Jtf;
      double F_val = F.jacobianProducts(JtJ, Jtf);
      double o[48] = {0};
      std::memcpy(o, JtJ.m, sizeof(JtJ.m));
      std::memcpy(o + 36, Jtf.v, sizeof(Jtf.v));
      o[43] = F_val;
      Matrix4d pose = F.pose();
      Vector6d dx;
      int result = sb_gn_step(o, last_error, epsilon, delta, pose.m, dx.v);
      F.increment(dx);
      Tk_ = F.pose();
      last_error = F_val;
      if (result == 0) break;
      ++k_;
    }
    return 0;
  }
  const Matrix4d& pose() const { return Tk_; }
  uint32_t iterationCount() const { return k_; }
  double residual() const { return last_error; }
  const std::vector<Matrix4d>& history() const { return history_; }

 protected:
  ContextPtr ctx_;
  double last_error{134567.00};
  uint32_t k_{0};
  Matrix4d Tk_;
  uint32_t maxIter{200};
  double epsilon{1e-10}, delta{1e-10};
  std::vector<Matrix4d> history_;
};

typedef sb_surfel Surfel;  // core/Surfel.h

/** core/SurfelMap.h */
class SurfelMap {
 public:
  explicit SurfelMap(const ContextPtr& ctx) : ctx_(ctx) {}
  void setParameters(const ParameterList& params) { ctx_->setParameters(params); }
  /** colours are a display concern (SurfelMap::setColorMap feeds draw_surfels.*): accepted and ignored */
  template <class ColorMap>
  void setColorMap(const ColorMap&) {}
  void reset() { check(sb_reset(ctx_->get()), ctx_->get(), "SurfelMap::reset"); }
  /** managed submap tile cache (sb_set_tile_cache; no counterpart in the reference): host_surfels = UINT64_MAX for no
   * bound. Only while the cache is empty (after construction or reset). */
  void setTileCache(uint32_t pool_surfels, uint64_t host_surfels) {
    check(sb_set_tile_cache(ctx_->get(), pool_surfels, host_surfels), ctx_->get(), "SurfelMap::setTileCache");
  }
  sb_tile_cache_info tileCacheInfo() const {
    sb_tile_cache_info info;
    check(sb_get_tile_cache_info(ctx_->get(), &info), ctx_->get(), "SurfelMap::tileCacheInfo");
    return info;
  }
  void update(const Matrix4f& pose, Frame& frame) {
    check(sb_map_update(ctx_->get(), pose.m, frame.handle()), ctx_->get(), "SurfelMap::update");
  }
  void render(const Matrix4f& pose, Frame& frame, float confidence_threshold) { render(pose, pose, frame, confidence_threshold); }
  void render(const Matrix4f& pose_old, const Matrix4f& pose_new, Frame& frame, float confidence_threshold) {
    check(sb_map_render(ctx_->get(), pose_old.m, pose_new.m, confidence_threshold, frame.handle()), ctx_->get(),
          "SurfelMap::render");
    frame.valid = true;
  }
  void render_active(const Matrix4f& pose, float ct) { check(sb_map_render_active(ctx_->get(), pose.m, ct), ctx_->get(), "render_active"); }
  void render_inactive(const Matrix4f& pose, float ct) { check(sb_map_render_inactive(ctx_->get(), pose.m, ct), ctx_->get(), "render_inactive"); }
  void render_composed(const Matrix4f& pose_old, const Matrix4f& pose_new, float ct) {
    check(sb_map_render_composed(ctx_->get(), pose_old.m, pose_new.m, ct), ctx_->get(), "render_composed");
  }
  std::shared_ptr<Frame> oldMapFrame() { return borrowed(SB_FRAME_OLD); }
  std::shared_ptr<Frame> newMapFrame() { return borrowed(SB_FRAME_NEW); }
  std::shared_ptr<Frame> composedFrame() { return borrowed(SB_FRAME_COMPOSED); }
  uint32_t size() const {
    uint32_t n = 0;
    sb_map_size(ctx_->get(), &n);
    return n;
  }
  void updatePoses(const std::vector<Matrix4f>& poses) {
    std::vector<float> a(poses.size() * 16);
    for (size_t i = 0; i < poses.size(); ++i) std::memcpy(a.data() + 16 * i, poses[i].m, 64);
    check(sb_map_update_poses(ctx_->get(), a.data(), static_cast<uint32_t>(poses.size())), ctx_->get(), "updatePoses");
  }
  std::vector<Surfel> getAllSurfels() {
    std::vector<Surfel> s(size());
    uint32_t n = 0;
    check(sb_map_download(ctx_->get(), s.data(), static_cast<uint32_t>(s.size()), &n), ctx_->get(), "getAllSurfels");
    s.resize(n);
    return s;
  }

 private:
  std::shared_ptr<Frame> borrowed(int which) {
    sb_frame* f = nullptr;
    check(sb_map_frame(ctx_->get(), which, &f), ctx_->get(), "map frame");
    return std::make_shared<Frame>(ctx_, f);
  }
  ContextPtr ctx_;
};

/** core/SurfelMapping.h (loop closure / pose graph stay with the caller: see INTEGRATION.md) */
class SurfelMapping {
 public:
  typedef std::unordered_map<std::string, float> Stats;
  explicit SurfelMapping(const ParameterList& params, int device = 0)
      : ctx_(std::make_shared<Context>(params, device)), map_(std::make_shared<SurfelMap>(ctx_)) {}
  void setParameters(const ParameterList& params) { ctx_->setParameters(params); }
  /** managed submap tile cache: see SurfelMap::setTileCache */
  void setTileCache(uint32_t pool_surfels, uint64_t host_surfels) { map_->setTileCache(pool_surfels, host_surfels); }
  sb_tile_cache_info tileCacheInfo() const { return map_->tileCacheInfo(); }
  /** per-point deskewing of every scan (sb_set_deskew; no counterpart in the reference) */
  void setDeskew(const sb_deskew_params& d) { check(sb_set_deskew(ctx_->get(), &d), ctx_->get(), "SurfelMapping::setDeskew"); }
  sb_deskew_params getDeskew() const {
    sb_deskew_params d;
    check(sb_get_deskew(ctx_->get(), &d), ctx_->get(), "SurfelMapping::getDeskew");
    return d;
  }
  /** per-point label records of every following scan (sb_set_point_labels; DESIGN.md section 13) */
  void setPointLabels(bool on) { check(sb_set_point_labels(ctx_->get(), on ? 1 : 0), ctx_->get(), "SurfelMapping::setPointLabels"); }
  /** the records of the last scan, one per input point in input order (sb_get_point_labels) */
  void getPointLabels(std::vector<sb_point_label>& out) const {
    uint32_t n = 0;
    const int rc = sb_get_point_labels(ctx_->get(), nullptr, 0, &n, 0);
    if (rc != SB_OK && !(rc == SB_ERR_INVALID && n > 0)) check(rc, ctx_->get(), "SurfelMapping::getPointLabels");
    out.resize(n);
    check(sb_get_point_labels(ctx_->get(), out.data(), n, &n, 0), ctx_->get(), "SurfelMapping::getPointLabels");
  }
  void reset() {
    check(sb_reset(ctx_->get()), ctx_->get(), "SurfelMapping::reset");
    trajectory_.clear();
  }
  /** processScan(scan), SurfelMapping.cpp:175-210 */
  void processScan(const Laserscan& scan) {
    check(sb_process_scan(ctx_->get(), scan.points.data(), scan.labels_float.empty() ? nullptr : scan.labels_float.data(),
                          scan.labels_prob.empty() ? nullptr : scan.labels_prob.data(), scan.size(), 0),
          ctx_->get(), "SurfelMapping::processScan");
    trajectory_.push_back(getCurrentPose());
  }
  /** processScan with one sweep time per point (deskewing mode 1; host memory, scan.size() values) */
  void processScan(const Laserscan& scan, const std::vector<float>& times) {
    if (times.size() != scan.size()) throw std::invalid_argument("SurfelMapping::processScan: one time per point");
    check(sb_process_scan_timed(ctx_->get(), scan.points.data(),
                                scan.labels_float.empty() ? nullptr : scan.labels_float.data(),
                                scan.labels_prob.empty() ? nullptr : scan.labels_prob.data(), times.data(), scan.size(), 0),
          ctx_->get(), "SurfelMapping::processScan");
    trajectory_.push_back(getCurrentPose());
  }
  /** SurfelMapping.cpp:904-907 hands the KITTI calibration to the preprocessor, whose shaders never read it: accepted, unused */
  template <class Calibration>
  void setCalibration(const Calibration&) {}
  template <class ColorMap>
  void setColorMap(const ColorMap& c) { map_->setColorMap(c); }
  Matrix4d getLastPose() const {
    Matrix4d p;
    sb_get_last_pose(ctx_->get(), p.m);
    return p;
  }
  Frame::Ptr getOldSurfelMap() { return map_->oldMapFrame(); }  // SurfelMapping.h:73
  Frame::Ptr getNewSurfelMap() { return map_->newMapFrame(); }  // SurfelMapping.h:74
  /** "close-loops" (config/default.xml:71): loop-closure detection and verification, SurfelMapping::checkLoopClosure
   * (SurfelMapping.cpp:527-795), run by the library between updatePose() and updateMap(). The pose-graph optimisation
   * (gtsam, core/Posegraph.cpp) stays with the caller (INTEGRATION.md section 3): getLoopEdges() returns the odometry and
   * loop edges the reference feeds into gtsam, optimisationRequested() mirrors the reference's trigger (:658-663); feed
   * the optimised poses back with integrateLoopClosures() (:212-258) before the next processScan. */
  void enableLoopClosure(bool on, const sb_loop_params* lp = nullptr) {
    check(sb_set_loop_closure(ctx_->get(), on ? 1 : 0, lp), ctx_->get(), "SurfelMapping::enableLoopClosure");
  }
  sb_loop_info getLoopInfo() const {
    sb_loop_info li;
    sb_get_loop_info(ctx_->get(), &li);
    return li;
  }
  std::vector<sb_loop_edge> getLoopEdges() const {
    uint32_t n = 0;
    sb_get_loop_edges(ctx_->get(), nullptr, 0, &n);
    std::vector<sb_loop_edge> e(n);
    if (n) sb_get_loop_edges(ctx_->get(), e.data(), n, &n);
    return e;
  }
  bool foundLoopClosureCandidate() const { return getLoopInfo().found_candidate != 0; }  // SurfelMapping.h:88
  bool useLoopClosureCandidate() const { return getLoopInfo().use_candidate != 0; }      // SurfelMapping.h:89
  bool optimisationRequested() const { return getLoopInfo().optimisation_requested != 0; }
  /** SurfelMapping::integrateLoopClosures (:212-258) with the optimised poses of scans 0 .. poses.size()-1 (empty: the
   * graph's own poses); returns the number of poses written to the map's pose table, 0 if no request was pending */
  uint32_t integrateLoopClosures(const std::vector<Matrix4d>& poses = std::vector<Matrix4d>()) {
    std::vector<double> a(poses.size() * 16);
    for (size_t i = 0; i < poses.size(); ++i) std::memcpy(&a[16 * i], poses[i].m, 128);
    uint32_t n = 0;
    check(sb_integrate_loop_closures(ctx_->get(), poses.empty() ? nullptr : a.data(), static_cast<uint32_t>(poses.size()), &n),
          ctx_->get(), "SurfelMapping::integrateLoopClosures");
    return n;
  }
  /** SurfelMapping::setCurrentPose, SurfelMapping.h:66 */
  void setCurrentPose(const Matrix4d& pose) {
    check(sb_set_current_pose(ctx_->get(), pose.m), ctx_->get(), "SurfelMapping::setCurrentPose");
  }
  /** without a pose-graph optimiser attached the "optimized" poses are the odometry poses */
  std::vector<Matrix4d> getOptimizedPoses() const { return trajectory_; }
  uint32_t timestamp() const {
    uint32_t t = 0;
    sb_timestamp(ctx_->get(), &t);
    return t;
  }
  Matrix4d getCurrentPose() const {
    Matrix4d p;
    sb_get_pose(ctx_->get(), p.m);
    return p;
  }
  std::shared_ptr<SurfelMap> getMap() { return map_; }
  Frame::Ptr getCurrentFrame() { return slam_frame(SB_SLAM_CURRENT); }
  Frame::Ptr getLastFrame() { return slam_frame(SB_SLAM_LAST); }
  Frame::Ptr getCurrentModelFrame() { return slam_frame(SB_SLAM_CURRENT_MODEL); }
  Frame::Ptr getLastModelFrame() { return slam_frame(SB_SLAM_LAST_MODEL); }
  Stats getStatistics() const {  // keys of SurfelMapping::statistics_, SurfelMapping.cpp:183-207
    double s[16];
    sb_get_statistics(ctx_->get(), s);
    Stats st;
    st["num_iterations"] = static_cast<float>(s[0]);
    st["preprocessing-time"] = static_cast<float>(s[8]);
    st["icp-time"] = static_cast<float>(s[9]);
    st["mapping-time"] = static_cast<float>(s[10]);
    st["complete-time"] = static_cast<float>(s[11]);
    st["residual"] = static_cast<float>(s[1]);
    st["inlier"] = static_cast<float>(s[2]);
    st["outlier"] = static_cast<float>(s[3]);
    st["invalid"] = static_cast<float>(s[4]);
    st["surfels"] = static_cast<float>(s[7]);
    const sb_loop_info li = getLoopInfo();
    if (li.enabled) {  // the keys checkLoopClosure writes (SurfelMapping.cpp:784-788)
      st["residual_old"] = static_cast<float>(li.residual_old);
      st["loop_outlier_ratio"] = li.outlier_ratio;
      st["loop_valid_ratio"] = li.valid_ratio;
      st["loop_relative_error_all"] = li.rel_error;
    }
    return st;
  }
  const ContextPtr& context() const { return ctx_; }

  /** Checkpoint of the whole mapping session (sb_state_save; no counterpart in the reference, whose
   * Posegraph::save/load are empty stubs): loading it into a SurfelMapping of the same image size and continuing gives
   * the bits of an uninterrupted run. */
  std::vector<uint8_t> saveState() const {
    uint64_t n = 0;
    check(sb_state_size(ctx_->get(), &n), ctx_->get(), "SurfelMapping::saveState");
    std::vector<uint8_t> blob(static_cast<size_t>(n));
    check(sb_state_save(ctx_->get(), blob.data(), n, &n), ctx_->get(), "SurfelMapping::saveState");
    blob.resize(static_cast<size_t>(n));
    return blob;
  }
  /** Restores a saveState() checkpoint and the parameters it carries. The odometry list of this mirror
   * (getOptimizedPoses) restarts at the load. */
  void loadState(const std::vector<uint8_t>& blob) {
    check(sb_state_load(ctx_->get(), blob.empty() ? nullptr : blob.data(), blob.size()), ctx_->get(),
          "SurfelMapping::loadState");
    sb_params p;
    check(sb_get_params(ctx_->get(), &p), ctx_->get(), "SurfelMapping::loadState");
    ctx_->adoptParameters(ParameterList(p));
    trajectory_.clear();
  }
  /** file variants, in the spirit of the reference's storePoseGraph(filename) */
  void saveState(const std::string& filename) const {
    const std::vector<uint8_t> blob = saveState();
    FILE* f = std::fopen(filename.c_str(), "wb");
    if (!f) throw std::runtime_error("SurfelMapping::saveState: cannot open " + filename);
    const bool ok = std::fwrite(blob.data(), 1, blob.size(), f) == blob.size();
    if (std::fclose(f) != 0 || !ok) throw std::runtime_error("SurfelMapping::saveState: cannot write " + filename);
  }
  void loadState(const std::string& filename) {
    FILE* f = std::fopen(filename.c_str(), "rb");
    if (!f) throw std::runtime_error("SurfelMapping::loadState: cannot open " + filename);
    std::vector<uint8_t> blob;
    uint8_t buf[1 << 16];
    size_t k;
    while ((k = std::fread(buf, 1, sizeof(buf), f)) > 0) blob.insert(blob.end(), buf, buf + k);
    std::fclose(f);
    loadState(blob);
  }

 private:
  Frame::Ptr slam_frame(int which) {
    sb_frame* f = nullptr;
    check(sb_slam_frame(ctx_->get(), which, &f), ctx_->get(), "slam frame");
    return std::make_shared<Frame>(ctx_, f);
  }
  ContextPtr ctx_;
  std::shared_ptr<SurfelMap> map_;
  std::vector<Matrix4d> trajectory_;
};

}  // namespace suma

#endif  // SUMA_B200_HPP_
