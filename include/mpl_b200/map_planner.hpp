/*
 * map_planner.hpp — header-only C++ host layer that puts the reference's class surface back on top of the C ABI
 * (include/mplb.h): MPL::MapUtil<Dim>, Waypoint<Dim>, Primitive<Dim>, Trajectory<Dim>, MPL::MapPlanner<Dim>
 * (OccMapPlanner / VoxelMapPlanner), with the member names and argument meaning of
 *   motion_primitive_library/include/mpl_collision/map_util.h        (MapUtil)
 *   motion_primitive_library/include/mpl_basis/waypoint.h            (Waypoint, control flags)
 *   motion_primitive_library/include/mpl_basis/primitive.h:205-431   (Primitive: coefficient rows, evaluate)
 *   motion_primitive_library/include/mpl_basis/trajectory.h:42-57,277-292
 *   motion_primitive_library/include/mpl_planner/common/planner_base.h:18-345 and planner/map_planner.h:20-125
 * so that callers written against the reference (MPL/test/test_planner_2d.cpp, mpl_test_node/src/
 * map_planner_node.cpp) compile against this header with their planner calls unchanged.
 *
 * Vector types: when Eigen is available (a ROS site) define MPL_B200_USE_EIGEN before including this header and
 * Vecf<N>/Veci<N>/VecDf are the reference's Eigen aliases (data_type.h:49-75); otherwise a minimal fixed-size
 * array type with operator() and operator[] is used (this image has no Eigen).
 *
 * Everything numerical runs in libmplb.so on the GPU; there is no CPU fallback — failures surface as `false`
 * from plan() with the message of mplb_last_error() printed when the planner is verbose.
 */
#ifndef MPL_B200_MAP_PLANNER_HPP
#define MPL_B200_MAP_PLANNER_HPP

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <memory>
#include <vector>

#include "../mplb.h"

typedef double decimal_t; /* data_type.h:49 */

/* printf colour macros of data_type.h:14-41 (the reference's callers use them in their own messages) */
#ifndef ANSI_COLOR_RED
#define ANSI_COLOR_RED "\x1b[1;31m"
#endif
#ifndef ANSI_COLOR_GREEN
#define ANSI_COLOR_GREEN "\x1b[1;32m"
#endif
#ifndef ANSI_COLOR_YELLOW
#define ANSI_COLOR_YELLOW "\x1b[1;33m"
#endif
#ifndef ANSI_COLOR_BLUE
#define ANSI_COLOR_BLUE "\x1b[1;34m"
#endif
#ifndef ANSI_COLOR_MAGENTA
#define ANSI_COLOR_MAGENTA "\x1b[1;35m"
#endif
#ifndef ANSI_COLOR_CYAN
#define ANSI_COLOR_CYAN "\x1b[1;36m"
#endif
#ifndef ANSI_COLOR_RESET
#define ANSI_COLOR_RESET "\x1b[0m"
#endif

#ifdef MPL_B200_USE_EIGEN
#include <Eigen/Geometry>
#include <Eigen/StdVector>
template <typename T>
using vec_E = std::vector<T, Eigen::aligned_allocator<T>>;
template <int N>
using Vecf = Eigen::Matrix<decimal_t, N, 1>;
template <int N>
using Veci = Eigen::Matrix<int, N, 1>;
typedef Eigen::Matrix<decimal_t, Eigen::Dynamic, 1> VecDf;
template <int M, int N>
using Matf = Eigen::Matrix<decimal_t, M, N>; /* data_type.h:77-101 */
typedef Matf<2, 2> Mat2f;
typedef Matf<3, 3> Mat3f;
typedef Matf<4, 4> Mat4f;
typedef Matf<6, 6> Mat6f;
typedef Vecf<6> Vec6f;
#else
template <typename T>
using vec_E = std::vector<T>;
template <typename T, int N>
struct mplb_small_vec {
  T v[N];
  mplb_small_vec() { for (int i = 0; i < N; i++) v[i] = T(0); }
  mplb_small_vec(T a, T b) { static_assert(N == 2, "2 components"); v[0] = a; v[1] = b; }
  mplb_small_vec(T a, T b, T c) { static_assert(N == 3, "3 components"); v[0] = a; v[1] = b; v[2] = c; }
  T &operator()(int i) { return v[i]; }
  const T &operator()(int i) const { return v[i]; }
  T &operator[](int i) { return v[i]; }
  const T &operator[](int i) const { return v[i]; }
  static mplb_small_vec Zero() { return mplb_small_vec(); }
  int size() const { return N; }
};
template <int N>
using Vecf = mplb_small_vec<decimal_t, N>;
template <int N>
using Veci = mplb_small_vec<int, N>;
typedef std::vector<decimal_t> VecDf; /* control rows: size() and operator[] like the Eigen dynamic vector */
#endif
template <int N>
using vec_Vecf = vec_E<Vecf<N>>;
template <int N>
using vec_Veci = vec_E<Veci<N>>;
typedef Vecf<2> Vec2f;
typedef Vecf<3> Vec3f;
typedef Veci<2> Vec2i;
typedef Veci<3> Vec3i;
typedef vec_Vecf<2> vec_Vec2f; /* data_type.h:89-95 */
typedef vec_Vecf<3> vec_Vec3f;
typedef vec_Veci<2> vec_Vec2i;
typedef vec_Veci<3> vec_Vec3i;

namespace Control { /* control.h:10-20 */
enum Control { NONE = 0, VEL = 0b00001, ACC = 0b00011, JRK = 0b00111, SNP = 0b01111,
               VELxYAW = 0b10001, ACCxYAW = 0b10011, JRKxYAW = 0b10111, SNPxYAW = 0b11111 };
}

/* waypoint.h:22-58 */
template <int Dim>
struct Waypoint {
  Waypoint() : control(Control::NONE) {}
  Waypoint(Control::Control c) : control(c) {}
  Vecf<Dim> pos, vel, acc, jrk;
  decimal_t yaw{0};
  decimal_t t{0};
  union {
    struct {
      bool use_pos : 1;
      bool use_vel : 1;
      bool use_acc : 1;
      bool use_jrk : 1;
      bool use_yaw : 1;
    };
    Control::Control control : 5;
  };
  bool enable_t{false};
};
typedef Waypoint<2> Waypoint2D;
typedef Waypoint<3> Waypoint3D;

/* primitive.h:205-431 — per-axis coefficient rows (highest order first), rebuilt exactly like
 * env_base::forward_action (env_base.h:228-231) from (parent state, U[action], dt). */
template <int Dim>
class Primitive {
 public:
  Primitive() {}
  Primitive(const Waypoint<Dim> &p, const VecDf &u, decimal_t t) : t_(t), control_(p.control) {
    for (int i = 0; i < Dim; i++) {
      double *c = c_[i];
      for (int k = 0; k < 6; k++) c[k] = 0;
      switch ((int)control_ & 15) { /* primitive.h:35-52; the *xYAW variants share the base rows (primitive.h:236-253) */
        case Control::VEL: c[4] = u[i]; c[5] = p.pos(i); break;
        case Control::ACC: c[3] = u[i]; c[4] = p.vel(i); c[5] = p.pos(i); break;
        case Control::JRK: c[2] = u[i]; c[3] = p.acc(i); c[4] = p.vel(i); c[5] = p.pos(i); break;
        case Control::SNP: c[1] = u[i]; c[2] = p.jrk(i); c[3] = p.acc(i); c[4] = p.vel(i); c[5] = p.pos(i); break;
        default: break;
      }
    }
    for (int k = 0; k < 6; k++) cyaw_[k] = 0;
    if (((int)control_ & 16) && (int)u.size() > Dim) { cyaw_[4] = u[Dim]; cyaw_[5] = p.yaw; } /* pr_yaw_ = Primitive1D(p.yaw, u(Dim)) */
  }
  /* Primitive(cs, t, control), primitive.h:309-313: coefficient rows given directly (Dim rows, optionally a yaw row) */
  Primitive(const double *rows6, const double *yaw6, decimal_t t, Control::Control control) : t_(t), control_(control) {
    for (int i = 0; i < Dim; i++)
      for (int k = 0; k < 6; k++) c_[i][k] = rows6[i * 6 + k];
    for (int k = 0; k < 6; k++) cyaw_[k] = yaw6 ? yaw6[k] : 0;
  }
  decimal_t t() const { return t_; }
  Control::Control control() const { return control_; }
  const double *coeff(int k) const { return c_[k]; } /* float64[6] row of planning_ros_msgs/Primitive (cx, cy, cz) */
  const double *coeff_yaw() const { return cyaw_; }  /* the cyaw row (primitive.h:346-347) */
  Waypoint<Dim> evaluate(decimal_t t) const { /* primitive.h:128-145,321-331 */
    Waypoint<Dim> p(control_);
    for (int k = 0; k < Dim; k++) {
      const double *c = c_[k];
      const double t2 = t * t, t3 = t2 * t, t4 = t3 * t, t5 = t4 * t;
      p.pos(k) = c[0] / 120 * t5 + c[1] / 24 * t4 + c[2] / 6 * t3 + c[3] / 2 * t * t + c[4] * t + c[5];
      p.vel(k) = c[0] / 24 * t4 + c[1] / 6 * t3 + c[2] / 2 * t * t + c[3] * t + c[4];
      p.acc(k) = c[0] / 6 * t3 + c[1] / 2 * t * t + c[2] * t + c[3];
      p.jrk(k) = c[0] / 2 * t * t + c[1] * t + c[2];
    }
    if (p.use_yaw) { /* primitive.h:328 with normalize_angle (math.h:15-19) */
      const double *c = cyaw_; /* Primitive1D::p, primitive.h:128-131 (a planner's yaw row has only c[4], c[5]) */
      const double t2 = t * t, t3 = t2 * t, t4 = t3 * t, t5 = t4 * t;
      decimal_t a = c[0] / 120 * t5 + c[1] / 24 * t4 + c[2] / 6 * t3 + c[3] / 2 * t * t + c[4] * t + c[5];
      while (a > M_PI) a -= 2.0 * M_PI;
      while (a < -M_PI) a += 2.0 * M_PI;
      p.yaw = a;
    }
    return p;
  }
  decimal_t J(const Control::Control &control) const { /* primitive.h:92-122 (full rows), summed over the axes :403-407 */
    decimal_t j = 0;
    const double t = t_;
    auto pw = [](double x, int n) { double r = 1; while (n-- > 0) r *= x; return r; }; /* math.h:197-203 */
    for (int k = 0; k < Dim; k++) {
      const double *c = c_[k];
      const int base = (int)control & 15; /* the yaw variants share the branch */
      if (base == Control::VEL)
        j += c[0] * c[0] / 5184 * pw(t, 9) + c[0] * c[1] / 576 * pw(t, 8) + (c[1] * c[1] / 252 + c[0] * c[2] / 168) * pw(t, 7) +
             (c[0] * c[3] / 72 + c[1] * c[2] / 36) * pw(t, 6) + (c[2] * c[2] / 20 + c[0] * c[4] / 60 + c[1] * c[3] / 15) * pw(t, 5) +
             (c[2] * c[3] / 4 + c[1] * c[4] / 12) * pw(t, 4) + (c[3] * c[3] / 3 + c[2] * c[4] / 3) * pw(t, 3) + c[3] * c[4] * t * t +
             c[4] * c[4] * t;
      else if (base == Control::ACC)
        j += c[0] * c[0] / 252 * pw(t, 7) + c[0] * c[1] / 36 * pw(t, 6) + (c[1] * c[1] / 20 + c[0] * c[2] / 15) * pw(t, 5) +
             (c[0] * c[3] / 12 + c[1] * c[2] / 4) * pw(t, 4) + (c[2] * c[2] / 3 + c[1] * c[3] / 3) * pw(t, 3) + c[2] * c[3] * t * t +
             c[3] * c[3] * t;
      else if (base == Control::JRK)
        j += c[0] * c[0] / 20 * pw(t, 5) + c[0] * c[1] / 4 * pw(t, 4) + (c[1] * c[1] + c[0] * c[2]) / 3 * pw(t, 3) + c[1] * c[2] * t * t +
             c[2] * c[2] * t;
      else if (base == Control::SNP)
        j += c[0] * c[0] / 3 * pw(t, 3) + c[0] * c[1] * t * t + c[1] * c[1] * t;
    }
    return j;
  }

 private:
  decimal_t t_{0};
  Control::Control control_{Control::NONE};
  double c_[Dim][6];
  double cyaw_[6];
};
typedef Primitive<2> Primitive2D;
typedef Primitive<3> Primitive3D;

/* trajectory.h:42-57,250-254,277-292 */
/* trajectory.h:19-35 */
template <int Dim>
struct Command {
  Vecf<Dim> pos, vel, acc, jrk;
  decimal_t yaw{0}, yaw_dot{0}, t{0};
};
typedef Command<2> Command2D;
typedef Command<3> Command3D;

template <int Dim>
class Trajectory {
 public:
  Trajectory() : total_t_(0) {}
  Trajectory(const vec_E<Primitive<Dim>> &prs) : segs(prs) {
    taus.push_back(0);
    for (const auto &pr : prs) taus.push_back(pr.t() + taus.back());
    total_t_ = taus.back();
  }
  decimal_t getTotalTime() const { return total_t_; }
  vec_E<Primitive<Dim>> getPrimitives() const { return segs; }
  decimal_t J(const Control::Control &control) const {
    decimal_t j = 0;
    for (const auto &seg : segs) j += seg.J(control);
    return j;
  }
  vec_E<Waypoint<Dim>> getWaypoints() const {
    vec_E<Waypoint<Dim>> ws;
    if (segs.empty()) return ws;
    decimal_t t = 0;
    for (const auto &seg : segs) {
      ws.push_back(seg.evaluate(0));
      ws.back().t = t;
      t += seg.t();
    }
    ws.push_back(segs.back().evaluate(segs.back().t()));
    ws.back().t = t;
    return ws;
  }
  /* trajectory.h:95-135 without a time-scaling lambda (a planner's trajectory never carries one): position and its
   * derivatives, yaw and yaw rate at `time`, clamped to [0, total time] */
  bool evaluate(decimal_t time, Command<Dim> &p) const {
    decimal_t tau = time;
    if (tau < 0) tau = 0;
    if (tau > total_t_) tau = total_t_;
    for (size_t id = 0; id < segs.size(); id++) {
      if (tau >= taus[id] && tau <= taus[id + 1]) {
        tau -= taus[id];
        const Waypoint<Dim> w = segs[id].evaluate(tau);
        p.pos = w.pos; p.vel = w.vel; p.acc = w.acc; p.jrk = w.jrk;
        const double *cy = segs[id].coeff_yaw();
        decimal_t a = cy[4] * tau + cy[5];
        while (a > M_PI) a -= 2.0 * M_PI;
        while (a < -M_PI) a += 2.0 * M_PI;
        p.yaw = a;
        decimal_t b = cy[4];
        while (b > M_PI) b -= 2.0 * M_PI;
        while (b < -M_PI) b += 2.0 * M_PI;
        p.yaw_dot = b;
        p.t = time;
        return true;
      }
    }
    return false;
  }
  vec_E<Command<Dim>> sample(int N) const { /* trajectory.h:230-237 */
    vec_E<Command<Dim>> ps(N + 1);
    const decimal_t dt = total_t_ / N;
    for (int i = 0; i <= N; i++) evaluate(i * dt, ps[i]);
    return ps;
  }
  vec_E<Primitive<Dim>> segs;
  std::vector<decimal_t> taus;

 private:
  decimal_t total_t_;
};
typedef Trajectory<2> Trajectory2D;
typedef Trajectory<3> Trajectory3D;

namespace MPL {

typedef std::vector<signed char> Tmap; /* map_util.h:14 */

/* map_util.h:20-314 — the grid lives on the GPU; getters read it back. */
template <int Dim>
class MapUtil {
 public:
  MapUtil() {}
  ~MapUtil() { if (h_) mplb_map_destroy(h_); }
  MapUtil(const MapUtil &) = delete;
  MapUtil &operator=(const MapUtil &) = delete;

  void setMap(const Vecf<Dim> &ori, const Veci<Dim> &dim, const Tmap &map, decimal_t res) { /* map_util.h:84-90 */
    if (h_) { /* same geometry (the replanner's getMap / edit / setMap, map_replanner_node.cpp:181-196): new cells in place, so
                 that planners sharing this MapUtil keep seeing it, as they do through the reference's shared_ptr */
      bool same = res == res_;
      for (int i = 0; i < Dim; i++) same = same && dim(i) == dim_(i) && ori(i) == origin_d_(i);
      if (same) {
        if (mplb_map_set_data(h_, reinterpret_cast<const int8_t *>(map.data())) != MPLB_OK) std::printf("[MapUtil] setMap failed: %s\n", mplb_last_error());
        return;
      }
      mplb_map_destroy(h_);
      h_ = nullptr;
    }
    int32_t nd[3] = {1, 1, 1};
    double o[3] = {0, 0, 0};
    for (int i = 0; i < Dim; i++) { nd[i] = dim(i); o[i] = ori(i); }
    dim_ = dim; origin_d_ = ori; res_ = res;
    if (mplb_map_create(Dim, nd, o, res, reinterpret_cast<const int8_t *>(map.data()), &h_) != MPLB_OK)
      std::printf("[MapUtil] setMap failed: %s\n", mplb_last_error());
  }
  void freeUnknown() { if (h_) mplb_map_free_unknown(h_); }                               /* map_util.h:259-276 */
  void dilate(const vec_Veci<Dim> &dilate_neighbor) {                                      /* map_util.h:221-257 */
    std::vector<int32_t> ns;
    for (const auto &it : dilate_neighbor) for (int i = 0; i < Dim; i++) ns.push_back(it(i));
    if (h_) mplb_map_dilate(h_, ns.data(), (int)dilate_neighbor.size());
  }
  Tmap getMap() {                                                                          /* map_util.h:25 */
    size_t n = 1;
    for (int i = 0; i < Dim; i++) n *= (size_t)dim_(i);
    Tmap m(n);
    if (h_) mplb_map_get_data(h_, reinterpret_cast<int8_t *>(m.data()), n);
    return m;
  }
  decimal_t getRes() { return res_; }
  Veci<Dim> getDim() { return dim_; }
  Vecf<Dim> getOrigin() { return origin_d_; }
  Veci<Dim> floatToInt(const Vecf<Dim> &pt) { /* map_util.h:103-108 */
    Veci<Dim> pn;
    for (int i = 0; i < Dim; i++) pn(i) = (int)std::round((pt(i) - origin_d_(i)) / res_ - 0.5);
    return pn;
  }
  Vecf<Dim> intToFloat(const Veci<Dim> &pn) { /* map_util.h:110-114 */
    Vecf<Dim> p;
    for (int i = 0; i < Dim; i++) p(i) = (pn(i) + 0.5) * res_ + origin_d_(i);
    return p;
  }
  bool isOutside(const Veci<Dim> &pn) { /* map_util.h:51-55 */
    for (int i = 0; i < Dim; i++) if (pn(i) < 0 || pn(i) >= dim_(i)) return true;
    return false;
  }
  vec_Vecf<Dim> getCloud() { /* map_util.h:137-162: centres of the occupied cells, x outermost */
    vec_Vecf<Dim> cloud;
    const Tmap m = getMap();
    const int nz = Dim == 3 ? dim_(Dim - 1) : 1;
    Veci<Dim> n;
    for (int x = 0; x < dim_(0); x++)
      for (int y = 0; y < dim_(1); y++)
        for (int z = 0; z < nz; z++) {
          n(0) = x; n(1) = y;
          if (Dim == 3) n(Dim - 1) = z;
          if (m[(size_t)x + (size_t)dim_(0) * y + (size_t)dim_(0) * dim_(1) * z] == 100) cloud.push_back(intToFloat(n));
        }
    return cloud;
  }
  vec_Veci<Dim> rayTrace(const Vecf<Dim> &pt1, const Vecf<Dim> &pt2) { /* map_util.h:117-134 */
    vec_Veci<Dim> pns;
    decimal_t q = 0;
    Vecf<Dim> diff;
    for (int i = 0; i < Dim; i++) { diff(i) = pt2(i) - pt1(i); q = std::max(q, std::abs(diff(i) / res_)); }
    const int max_diff = (int)(q / 0.8);
    const decimal_t s = 1.0 / max_diff;
    Veci<Dim> prev;
    for (int i = 0; i < Dim; i++) prev(i) = -1;
    for (int n = 1; n < max_diff; n++) {
      Vecf<Dim> pt;
      for (int i = 0; i < Dim; i++) pt(i) = pt1(i) + diff(i) * s * n;
      const Veci<Dim> pn = floatToInt(pt);
      if (isOutside(pn)) break;
      bool same = true;
      for (int i = 0; i < Dim; i++) same = same && pn(i) == prev(i);
      if (!same) pns.push_back(pn);
      prev = pn;
    }
    return pns;
  }
  /* rayTrace of many rays and the replanner node's cell selection on the GPU (mplb_map_trace_cells): for every traced cell pn
   * of ray i (p1s[i] -> p2s[i]) and every offset of `ns` (empty: the offset 0), pn + ns[k] when `select` (MPLB_TRACE_ALL /
   * _FREE / _OCCUPIED) keeps it; `offsets` (may be NULL) receives n + 1 entries, ray i owning cells offsets[i] .. offsets[i+1]-1 */
  vec_Veci<Dim> traceCells(const vec_Vecf<Dim> &p1s, const vec_Vecf<Dim> &p2s, const vec_Veci<Dim> &ns = vec_Veci<Dim>(),
                           int select = MPLB_TRACE_ALL, std::vector<int64_t> *offsets = nullptr) {
    vec_Veci<Dim> out;
    const size_t n = std::min(p1s.size(), p2s.size());
    std::vector<double> a(n * 3, 0.0), b(n * 3, 0.0);
    std::vector<int32_t> s3(ns.size() * 3, 0);
    for (size_t i = 0; i < n; i++) for (int k = 0; k < Dim; k++) { a[i * 3 + k] = p1s[i](k); b[i * 3 + k] = p2s[i](k); }
    for (size_t i = 0; i < ns.size(); i++) for (int k = 0; k < Dim; k++) s3[i * 3 + k] = ns[i](k);
    std::vector<int64_t> off(n + 1, 0);
    if (!h_) return out;
    const int64_t total = mplb_map_trace_cells(h_, a.data(), b.data(), (int)n, s3.empty() ? nullptr : s3.data(), (int)ns.size(), select,
                                               nullptr, 0, off.data());
    if (total < 0) { std::printf("[MapUtil] traceCells failed: %s\n", mplb_last_error()); return out; }
    std::vector<int32_t> c3((size_t)(total > 0 ? total : 1) * 3);
    mplb_map_trace_cells(h_, a.data(), b.data(), (int)n, s3.empty() ? nullptr : s3.data(), (int)ns.size(), select, c3.data(), total,
                         off.data());
    for (int64_t r = 0; r < total; r++) { Veci<Dim> pn; for (int k = 0; k < Dim; k++) pn(k) = c3[r * 3 + k]; out.push_back(pn); }
    if (offsets) *offsets = off;
    return out;
  }
  /* isFree / isOccupied / isUnknown by coordinate (map_util.h:57-80): outside is none of them */
  bool isFree(const Veci<Dim> &pn) { const int v = cell(pn); return v >= 0 && v < 100; }
  bool isOccupied(const Veci<Dim> &pn) { return cell(pn) == 100; }
  bool isUnknown(const Veci<Dim> &pn) { return cell(pn) == -1; }
  mplb_map *handle() const { return h_; }

 private:
  int cell(const Veci<Dim> &pn) {
    int32_t c[3] = {0, 0, 0}, v = std::numeric_limits<int32_t>::min();
    for (int i = 0; i < Dim; i++) c[i] = pn(i);
    if (h_) mplb_map_get_cells(h_, c, 1, &v);
    return v;
  }
  mplb_map *h_ = nullptr;
  decimal_t res_ = 0;
  Vecf<Dim> origin_d_;
  Veci<Dim> dim_;
};
typedef MapUtil<2> OccMapUtil;
typedef MapUtil<3> VoxelMapUtil;

/* planner_base.h:18-345 + map_planner.h:20-125 */
template <int Dim>
class MapPlanner {
 public:
  typedef Waypoint<Dim> Coord;
  MapPlanner(bool verbose = false) : planner_verbose_(verbose) {
    if (mplb_planner_create(Dim, verbose ? 1 : 0, &h_) != MPLB_OK) std::printf("[MapPlanner] %s\n", mplb_last_error());
  }
  ~MapPlanner() { if (h_) mplb_planner_destroy(h_); }
  MapPlanner(const MapPlanner &) = delete;
  MapPlanner &operator=(const MapPlanner &) = delete;

  void setMapUtil(const std::shared_ptr<MapUtil<Dim>> &map_util) { /* map_planner.cpp:14-18 */
    map_util_ = map_util;
    bound_map_ = map_util ? map_util->handle() : nullptr;
    if (h_ && map_util && mplb_planner_set_map(h_, map_util->handle()) != MPLB_OK) report();
  }
  bool initialized() { return initialized_; }
  void setVmax(decimal_t v) { set(MPLB_V_MAX, v); }
  void setAmax(decimal_t a) { set(MPLB_A_MAX, a); }
  void setJmax(decimal_t j) { set(MPLB_J_MAX, j); }
  void setYawmax(decimal_t yaw) { set(MPLB_YAW_MAX, yaw); }   /* planner_base.h:197 */
  void setWyaw(decimal_t w) { set(MPLB_WYAW, w); }             /* planner_base.h:221 */
  void setTmax(decimal_t t) { set(MPLB_T_MAX, t); }
  void setDt(decimal_t dt) { dt_ = dt; set(MPLB_DT, dt); }
  void setW(decimal_t w) { set(MPLB_W, w); }
  void setEpsilon(decimal_t eps) { set(MPLB_EPSILON, eps); }
  void setMaxNum(int num) { set(MPLB_MAX_NUM, num); }
  void setHeurIgnoreDynamics(bool ignore) { /* planner_base.h:233: only the default (true) is on this path */
    if (!ignore) std::printf("[MapPlanner] heur_ignore_dynamics = false is not supported (env_base.h:67-211 needs a polynomial root finder)\n");
  }
  void reset() { /* planner_base.h:164-167 */
    traj_ = Trajectory<Dim>(); initialized_ = false; last_ = mplb_result{};
    if (h_) mplb_planner_reset(h_);
  }
  /* ---- LPA* (planner_base.h:155,170-176; map_planner.h:74-87; caller: mpl_test_node/src/map_replanner_node.cpp) */
  void setLPAstar(bool use_lpastar) { /* planner_base.h:170-176 */
    use_lpastar_ = use_lpastar;
    if (h_ && mplb_planner_set_lpastar(h_, use_lpastar ? 1 : 0) != MPLB_OK) report();
    if (use_lpastar_) std::printf("[PlannerBase] use Lifelong Planning A*\n");
    else std::printf("[PlannerBase] use normal A*\n");
  }
  void getSubStateSpace(int time_step) { if (h_ && mplb_get_sub_state_space(h_, time_step) < 0) report(); } /* planner_base.h:155 */
  vec_Vecf<Dim> getLinkedNodes() const { /* map_planner.cpp:125-158 */
    vec_Vecf<Dim> pts;
    const int n = h_ ? mplb_get_linked_nodes(h_, nullptr, 0) : 0;
    if (n <= 0) return pts;
    std::vector<double> p3((size_t)n * 3);
    mplb_get_linked_nodes(h_, p3.data(), n);
    for (int i = 0; i < n; i++) { Vecf<Dim> q; for (int k = 0; k < Dim; k++) q(k) = p3[(size_t)i * 3 + k]; pts.push_back(q); }
    return pts;
  }
  void updateBlockedNodes(const vec_Veci<Dim> &blocked_pns) { update_nodes(blocked_pns, true); }  /* map_planner.cpp:160-171 */
  void updateClearedNodes(const vec_Veci<Dim> &cleared_pns) { update_nodes(cleared_pns, false); } /* map_planner.cpp:173-185 */
  void setPriorTrajectory(const Trajectory<Dim> &traj) { /* planner_base.h:249-252 */
    const auto &segs = traj.segs;
    std::vector<double> cs(segs.size() * 24, 0.0), ts(segs.size(), 0.0);
    for (size_t i = 0; i < segs.size(); i++) {
      for (int k = 0; k < Dim; k++) for (int q = 0; q < 6; q++) cs[i * 24 + k * 6 + q] = segs[i].coeff(k)[q];
      for (int q = 0; q < 6; q++) cs[i * 24 + 18 + q] = segs[i].coeff_yaw()[q];
      ts[i] = segs[i].t();
    }
    const int ctl = segs.empty() ? 0 : (int)segs.back().control();
    if (h_ && mplb_planner_set_prior_trajectory(h_, (int)segs.size(), cs.data(), ts.data(), ctl) != MPLB_OK) report();
  }
  void setTol(decimal_t tol_pos, decimal_t tol_vel = -1, decimal_t tol_acc = -1) { /* planner_base.h:255-265 */
    set(MPLB_TOL_POS, tol_pos); set(MPLB_TOL_VEL, tol_vel); set(MPLB_TOL_ACC, tol_acc);
  }
  void setU(const vec_E<VecDf> &U) { /* planner_base.h:246 */
    U_ = U;
    const int udim = (!U.empty() && (int)U[0].size() > Dim) ? Dim + 1 : Dim; /* Dim + 1: last entry is the yaw rate (primitive.h:217) */
    std::vector<double> flat;
    for (const auto &u : U) for (int k = 0; k < udim; k++) flat.push_back(u[k]);
    if (h_ && mplb_planner_set_controls(h_, flat.data(), (int)U.size(), udim) != MPLB_OK) report();
  }

  /* planner_base.h:275-325 */
  bool plan(const Coord &start, const Coord &goal) {
    mplb_waypoint s = to_c(start), g = to_c(goal);
    control_ = start.control;
    if (h_ && map_util_ && map_util_->handle() != bound_map_) setMapUtil(map_util_); /* the MapUtil re-created its grid since */
    /* traj_ is rewritten only where the reference writes it: recoverTraj's success or failure (graph_search.h:447-451);
     * start-not-free (planner_base.h:283-287), start-is-goal (graph_search.h:44), MaxExpandStep and the empty queue
     * (graph_search.h:149-161) leave the previous trajectory in place. */
    if (!h_ || mplb_plan(h_, &s, &g, &last_) != MPLB_OK) { report(); traj_cost_ = std::numeric_limits<decimal_t>::infinity(); return false; }
    return planned();
  }

  /* ---- fleets: one library call per replan step for many LPA* replanners (mplb_lpa_plan_batch and the mplb_lpa_*_batch
   * calls).  Entry i leaves planners[i] exactly as the single member would; a call returns false (message printed by the first
   * planner when it is verbose) when the library refused it, in which case no planner changed. */
  static bool planLPABatch(const std::vector<MapPlanner *> &planners, const vec_E<Coord> &starts, const vec_E<Coord> &goals,
                           std::vector<bool> *ok = nullptr) {
    const size_t n = planners.size();
    std::vector<mplb_planner *> h(n);
    std::vector<mplb_waypoint> s(n), g(n);
    std::vector<mplb_result> res(n > 0 ? n : 1);
    for (size_t i = 0; i < n; i++) {
      MapPlanner *p = planners[i];
      if (p->h_ && p->map_util_ && p->map_util_->handle() != p->bound_map_) p->setMapUtil(p->map_util_);
      h[i] = p->h_; s[i] = to_c(starts[i]); g[i] = to_c(goals[i]);
    }
    if (mplb_lpa_plan_batch(h.data(), (int)n, s.data(), g.data(), res.data()) != MPLB_OK) return batch_failed(planners);
    if (ok) ok->assign(n, false);
    for (size_t i = 0; i < n; i++) {
      MapPlanner *p = planners[i];
      p->control_ = starts[i].control;
      p->last_ = res[i];
      const bool r = p->planned();
      if (ok) (*ok)[i] = r;
    }
    return true;
  }
  static std::vector<vec_Vecf<Dim>> getLinkedNodesBatch(const std::vector<MapPlanner *> &planners) {
    const size_t n = planners.size();
    std::vector<vec_Vecf<Dim>> out(n);
    std::vector<mplb_planner *> h = handles(planners);
    std::vector<int32_t> counts(n > 0 ? n : 1, 0);
    if (mplb_lpa_get_linked_nodes_batch(h.data(), (int)n, counts.data(), nullptr, 0) != MPLB_OK) { batch_failed(planners); return out; }
    int64_t total = 0;
    for (size_t i = 0; i < n; i++) total += counts[i];
    std::vector<double> p3((size_t)(total > 0 ? total : 1) * 3);
    if (mplb_lpa_get_linked_nodes_batch(h.data(), (int)n, counts.data(), p3.data(), total) != MPLB_OK) { batch_failed(planners); return out; }
    size_t r = 0;
    for (size_t i = 0; i < n; i++)
      for (int j = 0; j < counts[i]; j++, r++) { Vecf<Dim> q; for (int k = 0; k < Dim; k++) q(k) = p3[r * 3 + k]; out[i].push_back(q); }
    return out;
  }
  static bool updateBlockedNodesBatch(const std::vector<MapPlanner *> &planners, const std::vector<vec_Veci<Dim>> &cells) {
    return update_batch(planners, cells, true);
  }
  static bool updateClearedNodesBatch(const std::vector<MapPlanner *> &planners, const std::vector<vec_Veci<Dim>> &cells) {
    return update_batch(planners, cells, false);
  }
  static bool getSubStateSpaceBatch(const std::vector<MapPlanner *> &planners, const std::vector<int> &time_steps) {
    const size_t n = planners.size();
    std::vector<mplb_planner *> h = handles(planners);
    std::vector<int32_t> ts(time_steps.begin(), time_steps.end()), sizes(n > 0 ? n : 1, 0);
    if (ts.empty()) ts.push_back(0);
    return mplb_lpa_sub_state_space_batch(h.data(), (int)n, ts.data(), sizes.data()) == MPLB_OK || batch_failed(planners);
  }

  /* ---- the cycle's output on the device (mplb.h: mplb_lpa_plan_batch_device and the calls after it).  Buffers are device
   * pointers on the planners' device, `stream` a cudaStream_t (NULL = default); each call returns after its work completed.
   * planLPABatchDevice leaves the library's retained trajectory as plan() does (getActions / getSegStates), but not this
   * object's last_ / traj_ / traj_cost_: nothing is read back. */
  static bool planLPABatchDevice(const std::vector<MapPlanner *> &planners, const void *d_starts, const void *d_goals, void *d_results,
                                 void *d_actions, void *d_seg_states, int max_seg, void *stream = nullptr) {
    std::vector<mplb_planner *> h = bound_handles(planners);
    return mplb_lpa_plan_batch_device(h.data(), (int)planners.size(), d_starts, d_goals, d_results, d_actions, d_seg_states, max_seg,
                                      stream) == MPLB_OK || batch_failed(planners);
  }
  /* getTraj().getWaypoints()[d_index[i]] of plan i (the replanner node's next start), d_ok[i] = 0 where there is none */
  static bool trajectoryWaypointsBatch(const std::vector<MapPlanner *> &planners, const void *d_results, const void *d_actions,
                                       const void *d_seg_states, int max_seg, const void *d_index, void *d_waypoints, void *d_ok,
                                       void *stream = nullptr) {
    std::vector<mplb_planner *> h = handles(planners);
    return mplb_lpa_trajectory_waypoints_device(h.data(), (int)planners.size(), d_results, d_actions, d_seg_states, max_seg, d_index,
                                                d_waypoints, d_ok, stream) == MPLB_OK || batch_failed(planners);
  }
  /* toTrajectoryROSMsg + the wire bytes of every plan, plan i with planner i's own controls and dt */
  static bool serializeLPABatch(const std::vector<MapPlanner *> &planners, const void *d_results, const void *d_actions,
                                const void *d_seg_states, int max_seg, void *d_out, size_t stride, void *d_len, double z = 0.0,
                                const char *frame_id = "map", uint32_t seq = 0, uint32_t stamp_sec = 0, uint32_t stamp_nsec = 0,
                                void *stream = nullptr) {
    std::vector<mplb_planner *> h = handles(planners);
    return mplb_lpa_serialize_trajectories_device(h.data(), (int)planners.size(), d_results, d_actions, d_seg_states, max_seg, z, seq,
                                                  stamp_sec, stamp_nsec, frame_id, d_out, stride, d_len, stream) == MPLB_OK ||
           batch_failed(planners);
  }
  /* map_planner_node.cpp:216-227 for every plan (coefficient rows [n][max_seg][Dim + 1][6]); n_segs may be NULL */
  static bool refineLPABatch(const std::vector<MapPlanner *> &planners, const void *d_results, const void *d_actions,
                             const void *d_seg_states, int max_seg, void *d_coefs, std::vector<int32_t> *n_segs = nullptr,
                             int control = MPLB_CONTROL_JRK, int yaw_control = MPLB_CONTROL_VEL, void *stream = nullptr) {
    std::vector<mplb_planner *> h = handles(planners);
    std::vector<int32_t> ns(planners.size() > 0 ? planners.size() : 1, 0);
    const bool ok = mplb_lpa_refine_trajectories_device(h.data(), (int)planners.size(), d_results, d_actions, d_seg_states, max_seg,
                                                        control, yaw_control, d_coefs, ns.data(), stream) == MPLB_OK;
    if (ok && n_segs) n_segs->assign(ns.begin(), ns.begin() + planners.size());
    return ok || batch_failed(planners);
  }

  /* ---- the same fleet sharded over the ranks of `comm` (DESIGN.md section 6.1): `planners` are this rank's robots
   * rank, rank + N, ... of n_total.  planLPAFleet is planLPABatch on them followed by mplb_fleet_plan's gather: on `root`,
   * results / actions (may be NULL) receive every robot's record and first max_seg actions in robot order.  It is collective:
   * every rank calls it with the same n_total, max_seg and root.  The cycle's map edit is mplb_fleet_map_edit on
   * map_util_->handle() with the robots' device cell lists (INTEGRATION.md). */
  static bool planLPAFleet(mplb_comm *comm, const std::vector<MapPlanner *> &planners, int n_total, const vec_E<Coord> &starts,
                           const vec_E<Coord> &goals, std::vector<mplb_result> *results = nullptr,
                           std::vector<int32_t> *actions = nullptr, int max_seg = 0, int root = 0) {
    const size_t n = planners.size();
    std::vector<mplb_planner *> h(n > 0 ? n : 1, nullptr);
    std::vector<mplb_waypoint> s(n > 0 ? n : 1), g(n > 0 ? n : 1);
    for (size_t i = 0; i < n; i++) {
      MapPlanner *p = planners[i];
      if (p->h_ && p->map_util_ && p->map_util_->handle() != p->bound_map_) p->setMapUtil(p->map_util_);
      h[i] = p->h_; s[i] = to_c(starts[i]); g[i] = to_c(goals[i]);
    }
    const bool is_root = mplb_comm_rank(comm) == root;
    const size_t n_res = is_root ? (size_t)n_total : n;
    std::vector<mplb_result> res(n_res > 0 ? n_res : 1);
    std::vector<int32_t> acts(is_root && max_seg > 0 ? (size_t)n_total * max_seg : 1, -1);
    if (mplb_fleet_plan(comm, h.data(), (int)n, n_total, s.data(), g.data(), res.data(), acts.data(), max_seg, root) != MPLB_OK)
      return batch_failed(planners);
    const int N = mplb_comm_size(comm), r0 = mplb_comm_rank(comm);
    for (size_t i = 0; i < n; i++) { /* the root's records are in robot order, the others' in local order */
      MapPlanner *p = planners[i];
      p->control_ = starts[i].control;
      p->last_ = res[is_root ? (size_t)r0 + i * N : i];
      p->planned();
    }
    if (is_root && results) results->assign(res.begin(), res.begin() + n_total);
    if (is_root && actions && max_seg > 0) *actions = acts;
    return true;
  }

 private:
  /* plan()'s bookkeeping after the library planned into last_ */
  bool planned() {
    initialized_ = true;
    traj_cost_ = last_.cost;
    if (last_.status == MPLB_PLAN_OK) {
      std::vector<int32_t> acts(last_.n_seg > 0 ? last_.n_seg : 1);
      std::vector<double> st((size_t)(last_.n_seg > 0 ? last_.n_seg : 1) * 13);
      mplb_get_actions(h_, acts.data(), (int)acts.size());
      mplb_get_seg_states(h_, st.data(), (int)acts.size());
      vec_E<Primitive<Dim>> prs;
      for (int i = 0; i < last_.n_seg; i++) {
        Waypoint<Dim> w(control_);
        for (int k = 0; k < Dim; k++) { w.pos(k) = st[i * 13 + k]; w.vel(k) = st[i * 13 + 3 + k]; w.acc(k) = st[i * 13 + 6 + k]; w.jrk(k) = st[i * 13 + 9 + k]; }
        w.yaw = st[i * 13 + 12];
        prs.push_back(Primitive<Dim>(w, U_[acts[i]], dt_));
      }
      traj_ = Trajectory<Dim>(prs);
    } else if (last_.status == MPLB_PLAN_TRACEBACK_FAILED) traj_ = Trajectory<Dim>();
    return last_.status == MPLB_PLAN_OK || last_.status == MPLB_PLAN_START_IS_GOAL;
  }
  static std::vector<mplb_planner *> handles(const std::vector<MapPlanner *> &planners) {
    std::vector<mplb_planner *> h(planners.size() > 0 ? planners.size() : 1, nullptr);
    for (size_t i = 0; i < planners.size(); i++) h[i] = planners[i]->h_;
    return h;
  }
  static std::vector<mplb_planner *> bound_handles(const std::vector<MapPlanner *> &planners) { /* as planLPABatch binds the map */
    for (MapPlanner *p : planners)
      if (p->h_ && p->map_util_ && p->map_util_->handle() != p->bound_map_) p->setMapUtil(p->map_util_);
    return handles(planners);
  }
  static bool batch_failed(const std::vector<MapPlanner *> &planners) {
    if (!planners.empty()) planners[0]->report();
    return false;
  }
  static bool update_batch(const std::vector<MapPlanner *> &planners, const std::vector<vec_Veci<Dim>> &cells, bool blocked) {
    const size_t n = planners.size();
    std::vector<mplb_planner *> h = handles(planners);
    std::vector<int64_t> off(n + 1, 0);
    std::vector<int32_t> c3, visited(n > 0 ? n : 1, 0);
    for (size_t i = 0; i < n; i++) {
      for (const auto &pn : cells[i]) for (int k = 0; k < 3; k++) c3.push_back(k < Dim ? pn(k) : 0);
      off[i + 1] = off[i] + (int64_t)cells[i].size();
    }
    return mplb_lpa_update_nodes_batch(h.data(), (int)n, blocked ? 1 : 0, c3.empty() ? nullptr : c3.data(), off.data(),
                                       visited.data()) == MPLB_OK || batch_failed(planners);
  }

 public:

  Trajectory<Dim> getTraj() const { return traj_; }          /* planner_base.h:28 */
  decimal_t getTrajCost() const { return traj_cost_; }       /* planner_base.h:155 */
  int getExpandedNum() const { return last_.pops; }          /* planner_base.h:148 */
  vec_Vecf<Dim> getCloseSet() const { return use_lpastar_ ? lpa_points(0) : node_points(2, false); }     /* planner_base.h:84-91 */
  vec_Vecf<Dim> getOpenSet() const {                                       /* planner_base.h:77-81 */
    if (use_lpastar_) return lpa_points(1);
    std::vector<mplb_node> nodes = fetch_nodes();
    std::vector<int32_t> ids(last_.n_open > 0 ? last_.n_open : 1);
    mplb_get_open(h_, ids.data(), (int)ids.size());
    vec_Vecf<Dim> ps;
    for (int i = 0; i < last_.n_open; i++) ps.push_back(pos_of(nodes[ids[i]]));
    return ps;
  }
  vec_Vecf<Dim> getExpandedNodes() const {                                 /* planner_base.h:140, env_map.h:154 */
    if (use_lpastar_) return vec_Vecf<Dim>(); /* the per-call expansion log is kept for A* plans only */
    std::vector<mplb_node> nodes = fetch_nodes();
    std::vector<int32_t> ids(last_.pops > 0 ? last_.pops : 1);
    int n = mplb_get_pop_log(h_, ids.data(), (int)ids.size());
    vec_Vecf<Dim> ps;
    for (int i = 0; i < n; i++) ps.push_back(pos_of(nodes[ids[i]]));
    return ps;
  }
  /* planner_base.h:143-145 (env_map.h:166): finite-cost primitives of every expanded node, in expansion order, rebuilt
   * by running get_succ (mplb_expand) over the popped states; plain-map plans only. */
  vec_E<Primitive<Dim>> getExpandedEdges() const {
    vec_E<Primitive<Dim>> prs;
    if (!h_ || last_.pops <= 0 || U_.empty()) return prs;
    std::vector<mplb_node> nodes = fetch_nodes();
    std::vector<int32_t> ids(last_.pops);
    const int n = mplb_get_pop_log(h_, ids.data(), (int)ids.size());
    if (n <= 0) return prs;
    std::vector<mplb_waypoint> st(n);
    for (int i = 0; i < n; i++) {
      const mplb_node &nd = nodes[ids[i]];
      mplb_waypoint &w = st[i];
      std::memset(&w, 0, sizeof(w));
      for (int k = 0; k < 3; k++) { w.pos[k] = nd.state[k]; w.vel[k] = nd.state[3 + k]; w.acc[k] = nd.state[6 + k]; w.jrk[k] = nd.state[9 + k]; }
      w.yaw = nd.state[12];
      w.control = (int)control_;
    }
    std::vector<mplb_prim_trace> rows((size_t)n * U_.size());
    if (mplb_expand(h_, st.data(), n, rows.data()) != MPLB_OK) { report(); return prs; }
    for (int i = 0; i < n; i++)
      for (size_t a = 0; a < U_.size(); a++) {
        const mplb_prim_trace &r = rows[(size_t)i * U_.size() + a];
        if (r.verdict < 3 || std::isinf(r.cost)) continue;
        Waypoint<Dim> w(control_);
        for (int k = 0; k < Dim; k++) { w.pos(k) = st[i].pos[k]; w.vel(k) = st[i].vel[k]; w.acc(k) = st[i].acc[k]; w.jrk(k) = st[i].jrk[k]; }
        w.yaw = st[i].yaw;
        prs.push_back(Primitive<Dim>(w, U_[a], dt_));
      }
    return prs;
  }
  /* planner_base.h:30-74: in A* a predecessor record is appended exactly when an expanded node yields a finite-cost
   * successor (graph_search.h:81,100-102), so both are the set of getExpandedEdges (the reference lists them in hash-map order) */
  vec_E<Primitive<Dim>> getValidPrimitives() const { return getExpandedEdges(); }
  vec_E<Primitive<Dim>> getAllPrimitives() const { return getExpandedEdges(); }
  const mplb_result &result() const { return last_; }
  mplb_planner *handle() const { return h_; }

  /* ---- cost shaping: search region + potential map (map_planner.h:27-54,77-87; env_map.h:104-128) */
  void setSearchRadius(const Vecf<Dim> &radius) { search_radius_ = radius; }            /* map_planner.cpp:41-43 */
  void setPotentialRadius(const Vecf<Dim> &radius) { potential_radius_ = radius; }      /* map_planner.cpp:20-23 */
  void setPotentialMapRange(const Vecf<Dim> &range) { potential_map_range_ = range; }   /* map_planner.cpp:25-28 */
  void setPotentialWeight(decimal_t w) { set(MPLB_POTENTIAL_WEIGHT, w); }               /* map_planner.cpp:30-33 */
  void setGradientWeight(decimal_t w) { set(MPLB_GRADIENT_WEIGHT, w); }                 /* map_planner.cpp:35-38 */
  void setSearchRegion(const vec_Vecf<Dim> &path, bool dense = false) {                 /* map_planner.cpp:46-95 */
    std::vector<double> flat(path.size() * 3, 0.0);
    for (size_t i = 0; i < path.size(); i++) for (int k = 0; k < Dim; k++) flat[i * 3 + k] = path[i](k);
    double r[3] = {0, 0, 0};
    for (int k = 0; k < Dim; k++) r[k] = search_radius_(k);
    if (h_ && mplb_planner_set_search_region_path(h_, flat.data(), (int)path.size(), dense ? 1 : 0, r) != MPLB_OK) report();
  }
  vec_Vecf<Dim> getSearchRegion() const {                                               /* map_planner.cpp:97-122 */
    vec_Vecf<Dim> pts;
    if (!h_ || !map_util_) return pts;
    const int64_t n = mplb_planner_get_search_region(h_, nullptr, 0);
    if (n <= 0) return pts;
    std::vector<uint8_t> in_region((size_t)n);
    mplb_planner_get_search_region(h_, in_region.data(), in_region.size());
    const Veci<Dim> dim = map_util_->getDim();
    Veci<Dim> c;
    const int nz = Dim == 3 ? dim(Dim - 1) : 1;
    for (int x = 0; x < dim(0); x++)
      for (int y = 0; y < dim(1); y++)
        for (int z = 0; z < nz; z++) {
          c(0) = x; c(1) = y;
          if (Dim == 3) c(Dim - 1) = z;
          if (in_region[(size_t)x + (size_t)dim(0) * y + (size_t)dim(0) * dim(1) * z]) pts.push_back(map_util_->intToFloat(c));
        }
    return pts;
  }
  void updatePotentialMap(const Vecf<Dim> &pos) {                                       /* map_planner.cpp:327-391 */
    double p3[3] = {0, 0, 0}, r[3] = {0, 0, 0}, g[3] = {0, 0, 0};
    for (int k = 0; k < Dim; k++) { p3[k] = pos(k); r[k] = potential_radius_(k); g[k] = potential_map_range_(k); }
    if (h_ && mplb_planner_update_potential_map(h_, p3, r, g, pow_) != MPLB_OK) report();
  }
  bool iterativePlan(const Coord &start, const Coord &goal, const Trajectory<Dim> &raw_traj, int max_num) { /* map_planner.cpp:394-434 */
    const bool verbose = planner_verbose_;
    planner_verbose_ = false;
    traj_ = raw_traj;
    decimal_t prev_traj_cost = 0;
    int cnt = 0;
    while (cnt < max_num) {
      cnt++;
      vec_Vecf<Dim> path;
      for (const auto &w : traj_.getWaypoints()) path.push_back(w.pos);
      setSearchRegion(path, false);
      if (!plan(start, goal)) {
        if (verbose) std::printf("[MapPlanner] fails the [%d] plan!\n", cnt);
        planner_verbose_ = verbose;
        return false;
      }
      if (prev_traj_cost == traj_cost_) {
        if (verbose) std::printf("[MapPlanner] Converged after %d iterations! Trajectory cost: %f\n", cnt, traj_cost_);
        break;
      }
      prev_traj_cost = traj_cost_;
    }
    planner_verbose_ = verbose;
    return true;
  }

 protected:
  void set(int key, double v) { if (h_ && mplb_planner_set_param(h_, key, v) != MPLB_OK) report(); }
  void report() const { if (planner_verbose_) std::printf("[MapPlanner] %s\n", mplb_last_error()); }
  static mplb_waypoint to_c(const Coord &w) {
    mplb_waypoint c;
    for (int k = 0; k < 3; k++) { c.pos[k] = c.vel[k] = c.acc[k] = c.jrk[k] = 0; }
    for (int k = 0; k < Dim; k++) { c.pos[k] = w.pos(k); c.vel[k] = w.vel(k); c.acc[k] = w.acc(k); c.jrk[k] = w.jrk(k); }
    c.yaw = w.yaw; c.t = w.t; c.control = (int)w.control; c.enable_t = w.enable_t ? 1 : 0;
    return c;
  }
  std::vector<mplb_node> fetch_nodes() const {
    std::vector<mplb_node> nodes(last_.n_nodes > 0 ? last_.n_nodes : 1);
    mplb_get_nodes(h_, nodes.data(), (int)nodes.size());
    return nodes;
  }
  static Vecf<Dim> pos_of(const mplb_node &n) {
    Vecf<Dim> p;
    for (int k = 0; k < Dim; k++) p(k) = n.state[k];
    return p;
  }
  vec_Vecf<Dim> node_points(int flag, bool) const {
    std::vector<mplb_node> nodes = fetch_nodes();
    vec_Vecf<Dim> ps;
    for (int i = 0; i < last_.n_nodes; i++)
      if ((flag == 2 && nodes[i].closed) || (flag == 1 && nodes[i].opened)) ps.push_back(pos_of(nodes[i]));
    return ps;
  }

  /* LPA* state space through the dumps: which = 0 closed members of hm_ (planner_base.h:84-91), 1 = the open list */
  vec_Vecf<Dim> lpa_points(int which) const {
    vec_Vecf<Dim> ps;
    const int n = h_ ? mplb_lpa_get_nodes(h_, nullptr, 0) : 0;
    if (n <= 0) return ps;
    std::vector<mplb_lpa_node> nodes(n);
    mplb_lpa_get_nodes(h_, nodes.data(), n);
    for (const auto &nd : nodes)
      if ((which == 0 && nd.closed) || (which == 1 && nd.opened && !nd.closed)) { Vecf<Dim> q; for (int k = 0; k < Dim; k++) q(k) = nd.state[k]; ps.push_back(q); }
    return ps;
  }
  void update_nodes(const vec_Veci<Dim> &pns, bool blocked) {
    std::vector<int32_t> c3(pns.size() * 3, 0);
    for (size_t i = 0; i < pns.size(); i++) for (int k = 0; k < Dim; k++) c3[i * 3 + k] = pns[i](k);
    const int rc = blocked ? mplb_update_blocked_nodes(h_, c3.data(), (int)pns.size()) : mplb_update_cleared_nodes(h_, c3.data(), (int)pns.size());
    if (rc < 0) report();
  }
  bool use_lpastar_ = false;
  mplb_map *bound_map_ = nullptr;
  mplb_planner *h_ = nullptr;
  std::shared_ptr<MapUtil<Dim>> map_util_;
  vec_E<VecDf> U_;
  decimal_t dt_ = 1.0;
  Control::Control control_ = Control::NONE;
  Trajectory<Dim> traj_;
  decimal_t traj_cost_ = std::numeric_limits<decimal_t>::infinity();
  mplb_result last_{};
  bool initialized_ = false;
  bool planner_verbose_;
  Vecf<Dim> search_radius_ = zero_vec(), potential_radius_ = zero_vec(), potential_map_range_ = zero_vec(); /* map_planner.h:106-111 */
  decimal_t pow_ = 1.0;                                                                                     /* map_planner.h:113 */
  static Vecf<Dim> zero_vec() { Vecf<Dim> v; for (int k = 0; k < Dim; k++) v(k) = 0; return v; }
};
typedef MapPlanner<2> OccMapPlanner;   /* map_planner.h:122 */
typedef MapPlanner<3> VoxelMapPlanner; /* map_planner.h:125 */

}  // namespace MPL
#endif
