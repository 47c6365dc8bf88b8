/*
 * mpl_oracle.cpp — CPU ORACLE: restatement of the reference A* hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference) may load this.
 * The product (mpl_ros_b200/) never links or calls it.
 *
 * Every function cites the reference lines it follows.  Abbreviations (all under
 * /root/reference/motion_primitive_library/include/):
 *   pr = mpl_basis/primitive.h      wp = mpl_basis/waypoint.h     mt = mpl_basis/math.h
 *   mu = mpl_collision/map_util.h   eb = mpl_planner/common/env_base.h
 *   em = mpl_planner/env/env_map.h  gs = mpl_planner/common/graph_search.h
 *   ss = mpl_planner/common/state_space.h   pb = mpl_planner/common/planner_base.h
 *
 * Build: g++ -O2 -std=c++17 -ffp-contract=off (mirrors the reference's -O2, no -march, no
 * fast-math: MPL/CMakeLists.txt:5-8) — no FMA contraction, IEEE double everywhere.
 *
 * Arithmetic is written in the SAME operation order as the reference expressions (all six
 * polynomial terms, power() by repeated multiplication, division by res, std::round).
 *
 * Assumptions about absent third-party code (see mpl_oracle.h): Eigen >= 3.2 semantics for
 * `vec / scalar` (element-wise IEEE division) — only reached in rayTrace (mu:117-134);
 * Boost d_ary_heap sift rules as documented at struct Heap below.
 */
#include "mpl_oracle.h"

#include <pthread.h>
#include <sched.h>
#include <unistd.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

namespace {

const double kInf = std::numeric_limits<double>::infinity();

/* ------------------------------------------------------------------ control bits, control.h:10-20 */
enum { USE_POS = 1, USE_VEL = 2, USE_ACC = 4, USE_JRK = 8, USE_YAW = 16 };
enum { C_VEL = 1, C_ACC = 3, C_JRK = 7, C_SNP = 15 };

struct WP {  // waypoint.h:22-58
  double pos[3] = {0, 0, 0}, vel[3] = {0, 0, 0}, acc[3] = {0, 0, 0}, jrk[3] = {0, 0, 0};
  double yaw = 0, t = 0;
  int control = 0;
  bool enable_t = false;
};

WP from_c(const orc_waypoint &w) {
  WP r;
  for (int i = 0; i < 3; i++) { r.pos[i] = w.pos[i]; r.vel[i] = w.vel[i]; r.acc[i] = w.acc[i]; r.jrk[i] = w.jrk[i]; }
  r.yaw = w.yaw; r.t = w.t; r.control = w.control; r.enable_t = w.enable_t != 0;
  return r;
}

/* ------------------------------------------------------------------ lattice key, wp:92-125
 * The reference folds these ints through boost::hash_combine and compares the 64-bit results
 * (wp:132-135); we keep the int tuple itself (equivalent up to hash collisions).            */
struct Key {
  int32_t v[15];
  int32_t n = 0;
  bool operator==(const Key &o) const { return n == o.n && std::memcmp(v, o.v, sizeof(int32_t) * n) == 0; }
};

Key make_key(const WP &w, int dim) {
  Key k;
  std::memset(k.v, 0, sizeof(k.v));
  for (int i = 0; i < dim; i++) {
    if (w.control & USE_POS) k.v[k.n++] = (int)std::round(w.pos[i] / 0.01);
    if (w.control & USE_VEL) k.v[k.n++] = (int)std::round(w.vel[i] / 0.1);
    if (w.control & USE_ACC) k.v[k.n++] = (int)std::round(w.acc[i] / 0.1);
    if (w.control & USE_JRK) k.v[k.n++] = (int)std::round(w.jrk[i] / 0.1);
  }
  if (w.control & USE_YAW) k.v[k.n++] = (int)std::round(w.yaw / 0.1);
  if (w.enable_t) k.v[k.n++] = (int)std::round(w.t / 0.1);
  return k;
}

/* 64-bit mixing hash of the int tuple: shared definition with the CUDA side (mplb key hash),
 * used for pop_hash / closed_hash parity and as std::unordered_map hasher. */
uint64_t key_hash(const Key &k) {
  uint64_t h = 0x243F6A8885A308D3ull;
  for (int i = 0; i < k.n; i++) {
    h ^= (uint64_t)(uint32_t)k.v[i];
    h *= 0x9E3779B97F4A7C15ull;
    h ^= h >> 32;
  }
  h ^= h >> 30; h *= 0xBF58476D1CE4E5B9ull;
  h ^= h >> 27; h *= 0x94D049BB133111EBull;
  h ^= h >> 31;
  return h;
}
struct KeyHasher { size_t operator()(const Key &k) const { return (size_t)key_hash(k); } };

/* ------------------------------------------------------------------ math.h:197-205 */
double power(double t, int n) {
  double tn = 1;
  while (n > 0) { tn *= t; n--; }
  return tn;
}

/* math.h:117-131 restricted to what the grid path reaches (quartic/cubic never on ACC/JRK/SNP grids:
 * a = 0 always, b = c0/6 = 0 always because c0 = 0 for every control constructor pr:35-52). */
std::vector<double> solve4(double a, double b, double c, double d, double e) {
  std::vector<double> ts;
  if (a != 0 || b != 0) {
    std::fprintf(stderr, "oracle: quartic/cubic extrema not on the grid path (a=%g b=%g)\n", a, b);
    return ts;
  }
  if (c != 0) {  // quad, math.h:22-33
    double p = d * d - 4 * c * e;
    if (p < 0) return ts;
    ts.push_back((-d - std::sqrt(p)) / (2 * c));
    ts.push_back((-d + std::sqrt(p)) / (2 * c));
    return ts;
  } else if (d != 0) {
    ts.push_back(-e / d);
    return ts;
  }
  return ts;
}


/* ------------------------------------------------------------------ correctly rounded sin/cos for the yaw branch
 * The reference calls libm cos/sin (pr:520, em:125) whose last bit is not specified (glibc 2.39 differs from the
 * correctly rounded value on about 0.14 % of arguments, always by one ulp).  To give the yaw branch a reproducible
 * definition the oracle can evaluate both: trig_mode 0 = libm (the reference as built on this machine),
 * trig_mode 1 = correctly rounded via double-double arithmetic (what the CUDA path implements).  Constants from
 * tools/gen_trig_tables.py.  Accuracy about 2^-100 relative, i.e. the rounding is correct unless the true value lies
 * within 2^-100 of a rounding boundary. */
namespace crtrig {
static const double PIO2_1 = 0x1.921fb54442d18p+0, PIO2_2 = 0x1.1a62633145c07p-54, PIO2_3 = -0x1.f1976b7ed8fbcp-110;
static const double TWO_OVER_PI = 0x1.45f306dc9c883p-1;
/* 1/n! as double-double (hi, lo), n = 2..31 */
static const double INV_FACT[30][2] = {
  {0x1.0000000000000p-1, 0x0.0p+0}, /* 1/2! */
  {0x1.5555555555555p-3, 0x1.5555555555555p-57}, /* 1/3! */
  {0x1.5555555555555p-5, 0x1.5555555555555p-59}, /* 1/4! */
  {0x1.1111111111111p-7, 0x1.1111111111111p-63}, /* 1/5! */
  {0x1.6c16c16c16c17p-10, -0x1.f49f49f49f49fp-65}, /* 1/6! */
  {0x1.a01a01a01a01ap-13, 0x1.a01a01a01a01ap-73}, /* 1/7! */
  {0x1.a01a01a01a01ap-16, 0x1.a01a01a01a01ap-76}, /* 1/8! */
  {0x1.71de3a556c734p-19, -0x1.c154f8ddc6c00p-73}, /* 1/9! */
  {0x1.27e4fb7789f5cp-22, 0x1.cbbc05b4fa99ap-76}, /* 1/10! */
  {0x1.ae64567f544e4p-26, -0x1.c062e06d1f209p-80}, /* 1/11! */
  {0x1.1eed8eff8d898p-29, -0x1.2aec959e14c06p-83}, /* 1/12! */
  {0x1.6124613a86d09p-33, 0x1.f28e0cc748ebep-87}, /* 1/13! */
  {0x1.93974a8c07c9dp-37, 0x1.05d6f8a2efd1fp-92}, /* 1/14! */
  {0x1.ae7f3e733b81fp-41, 0x1.1d8656b0ee8cbp-97}, /* 1/15! */
  {0x1.ae7f3e733b81fp-45, 0x1.1d8656b0ee8cbp-101}, /* 1/16! */
  {0x1.952c77030ad4ap-49, 0x1.ac981465ddc6cp-103}, /* 1/17! */
  {0x1.6827863b97d97p-53, 0x1.eec01221a8b0bp-107}, /* 1/18! */
  {0x1.2f49b46814157p-57, 0x1.2650f61dbdcb4p-112}, /* 1/19! */
  {0x1.e542ba4020225p-62, 0x1.ea72b4afe3c2fp-120}, /* 1/20! */
  {0x1.71b8ef6dcf572p-66, -0x1.d043ae40c4647p-120}, /* 1/21! */
  {0x1.0ce396db7f853p-70, -0x1.aebcdbd20331cp-124}, /* 1/22! */
  {0x1.761b41316381ap-75, -0x1.3423c7d91404fp-130}, /* 1/23! */
  {0x1.f2cf01972f578p-80, -0x1.9ada5fcc1ab14p-135}, /* 1/24! */
  {0x1.3f3ccdd165fa9p-84, -0x1.58ddadf344487p-139}, /* 1/25! */
  {0x1.88e85fc6a4e5ap-89, -0x1.71c37ebd16540p-143}, /* 1/26! */
  {0x1.d1ab1c2dccea3p-94, 0x1.054d0c78aea14p-149}, /* 1/27! */
  {0x1.0a18a2635085dp-98, 0x1.b9e2e28e1aa54p-153}, /* 1/28! */
  {0x1.259f98b4358adp-103, 0x1.eaf8c39dd9bc5p-157}, /* 1/29! */
  {0x1.3932c5047d60ep-108, 0x1.832b7b530a627p-162}, /* 1/30! */
  {0x1.434d2e783f5bcp-113, 0x1.0b87b91be9affp-167}, /* 1/31! */
};

struct DD { double hi, lo; };
inline DD two_sum(double a, double b) { double s = a + b, bb = s - a; return {s, (a - (s - bb)) + (b - bb)}; }
inline DD quick_two_sum(double a, double b) { double s = a + b; return {s, b - (s - a)}; }
inline DD two_prod(double a, double b) { double p = a * b; return {p, std::fma(a, b, -p)}; }
inline DD dd_add(DD x, DD y) {
  DD s = two_sum(x.hi, y.hi), t = two_sum(x.lo, y.lo);
  s.lo += t.hi;
  s = quick_two_sum(s.hi, s.lo);
  s.lo += t.lo;
  return quick_two_sum(s.hi, s.lo);
}
inline DD dd_mul(DD x, DD y) {
  DD p = two_prod(x.hi, y.hi);
  p.lo += x.hi * y.lo + x.lo * y.hi;
  return quick_two_sum(p.hi, p.lo);
}
inline DD dd_neg(DD x) { return {-x.hi, -x.lo}; }

/* sin and cos of x for |x| < 2^20, each rounded to nearest. */
void sincos_cr(double x, double *sn, double *cs) {
  double kd = std::nearbyint(x * TWO_OVER_PI);
  long k = (long)kd;
  /* r = x - k*pi/2 with pi/2 = P1 + P2 + P3 (161 bits) */
  DD a = two_prod(kd, PIO2_1), b = two_prod(kd, PIO2_2), c = two_prod(kd, PIO2_3);
  DD r = two_sum(x, -a.hi);
  r = dd_add(r, {-a.lo, 0.0});
  r = dd_add(r, dd_neg(b));
  r = dd_add(r, dd_neg(c));
  DD r2 = dd_mul(r, r);
  /* sin r = r (1 - r2/3! + r2^2/5! - ...), cos r = 1 - r2/2! + r2^2/4! - ...  (Horner in r2, |r| <= pi/4) */
  DD ps = {INV_FACT[29][0], INV_FACT[29][1]}; /* 1/31! */
  for (int n = 29; n >= 3; n -= 2) {
    ps = dd_mul(ps, r2);
    DD cf = {INV_FACT[n - 2][0], INV_FACT[n - 2][1]};
    ps = dd_add(cf, dd_neg(ps));
  }
  ps = dd_mul(ps, r2);
  ps = dd_add({1.0, 0.0}, dd_neg(ps));
  DD s = dd_mul(ps, r);
  DD pc = {INV_FACT[28][0], INV_FACT[28][1]}; /* 1/30! */
  for (int n = 28; n >= 2; n -= 2) {
    pc = dd_mul(pc, r2);
    DD cf = {INV_FACT[n - 2][0], INV_FACT[n - 2][1]};
    pc = dd_add(cf, dd_neg(pc));
  }
  pc = dd_mul(pc, r2);
  DD cq = dd_add({1.0, 0.0}, dd_neg(pc));
  DD so, co;
  switch ((int)(((k % 4) + 4) % 4)) {
    case 0: so = s; co = cq; break;
    case 1: so = cq; co = dd_neg(s); break;
    case 2: so = dd_neg(s); co = dd_neg(cq); break;
    default: so = dd_neg(cq); co = s; break;
  }
  *sn = so.hi + so.lo;
  *cs = co.hi + co.lo;
}
}  // namespace crtrig

/* ------------------------------------------------------------------ Primitive1D, pr:21-198 */
struct Prim1D {
  double c[6] = {0, 0, 0, 0, 0, 0};
  double p(double t) const {  // pr:128-131
    return c[0] / 120 * power(t, 5) + c[1] / 24 * power(t, 4) + c[2] / 6 * power(t, 3) + c[3] / 2 * t * t + c[4] * t + c[5];
  }
  double v(double t) const {  // pr:134-137
    return c[0] / 24 * power(t, 4) + c[1] / 6 * power(t, 3) + c[2] / 2 * t * t + c[3] * t + c[4];
  }
  double a(double t) const {  // pr:140-142
    return c[0] / 6 * power(t, 3) + c[1] / 2 * t * t + c[2] * t + c[3];
  }
  double j(double t) const { return c[0] / 2 * t * t + c[1] * t + c[2]; }  // pr:145
  std::vector<double> extrema_v(double t) const {  // pr:152-162
    std::vector<double> roots = solve4(0, c[0] / 6, c[1] / 2, c[2], c[3]);
    std::vector<double> ts;
    for (double it : roots) {
      if (it > 0 && it < t) ts.push_back(it);
      else if (it >= t) break;
    }
    return ts;
  }
  std::vector<double> extrema_a(double t) const {  // pr:169-179
    std::vector<double> roots = solve4(0, 0, c[0] / 2, c[1], c[2]);
    std::vector<double> ts;
    for (double it : roots) {
      if (it > 0 && it < t) ts.push_back(it);
      else if (it >= t) break;
    }
    return ts;
  }
  std::vector<double> extrema_j(double t) const {  // pr:186-193
    std::vector<double> ts;
    if (c[0] != 0) {
      double t_sol = -c[1] * 2 / c[0];
      if (t_sol > 0 && t_sol < t) ts.push_back(t_sol);
    }
    return ts;
  }
  double J(double t, int control) const {  // pr:92-122 (yaw variants share the branch)
    int cc = control & 15;
    if (cc == C_VEL)
      return c[0] * c[0] / 5184 * power(t, 9) + c[0] * c[1] / 576 * power(t, 8) +
             (c[1] * c[1] / 252 + c[0] * c[2] / 168) * power(t, 7) + (c[0] * c[3] / 72 + c[1] * c[2] / 36) * power(t, 6) +
             (c[2] * c[2] / 20 + c[0] * c[4] / 60 + c[1] * c[3] / 15) * power(t, 5) +
             (c[2] * c[3] / 4 + c[1] * c[4] / 12) * power(t, 4) + (c[3] * c[3] / 3 + c[2] * c[4] / 3) * power(t, 3) +
             c[3] * c[4] * t * t + c[4] * c[4] * t;
    else if (cc == C_ACC)
      return c[0] * c[0] / 252 * power(t, 7) + c[0] * c[1] / 36 * power(t, 6) +
             (c[1] * c[1] / 20 + c[0] * c[2] / 15) * power(t, 5) + (c[0] * c[3] / 12 + c[1] * c[2] / 4) * power(t, 4) +
             (c[2] * c[2] / 3 + c[1] * c[3] / 3) * power(t, 3) + c[2] * c[3] * t * t + c[3] * c[3] * t;
    else if (cc == C_JRK)
      return c[0] * c[0] / 20 * power(t, 5) + c[0] * c[1] / 4 * power(t, 4) + (c[1] * c[1] + c[0] * c[2]) / 3 * power(t, 3) +
             c[1] * c[2] * t * t + c[2] * c[2] * t;
    else if (cc == C_SNP)
      return c[0] * c[0] / 3 * power(t, 3) + c[0] * c[1] * t * t + c[1] * c[1] * t;
    return 0;
  }
};

/* ------------------------------------------------------------------ Primitive<Dim>, pr:205-431 */
struct Prim {
  int dim = 3;
  double T = 0;
  int control = 0;
  Prim1D ax[3];
  Prim1D yawp;  // pr_yaw_, pr:430 (Primitive1D(p.yaw, u(Dim)), pr:36,242-253)

  Prim() {}
  Prim(const WP &p, const double *u, double t, int dim_) : dim(dim_), T(t), control(p.control) {  // pr:220-256
    int cc = control & 15;
    if (control & USE_YAW) { yawp.c[4] = u[dim_]; yawp.c[5] = p.yaw; }
    for (int i = 0; i < dim; i++) {
      double *c = ax[i].c;
      if (cc == C_SNP) { c[1] = u[i]; c[2] = p.jrk[i]; c[3] = p.acc[i]; c[4] = p.vel[i]; c[5] = p.pos[i]; }       // pr:50-52
      else if (cc == C_JRK) { c[2] = u[i]; c[3] = p.acc[i]; c[4] = p.vel[i]; c[5] = p.pos[i]; }                   // pr:44-46
      else if (cc == C_ACC) { c[3] = u[i]; c[4] = p.vel[i]; c[5] = p.pos[i]; }                                    // pr:40
      else if (cc == C_VEL) { c[4] = u[i]; c[5] = p.pos[i]; }                                                     // pr:36
    }
  }
  static double normalize_angle(double angle) {  // math.h:15-19
    while (angle > M_PI) angle -= 2.0 * M_PI;
    while (angle < -M_PI) angle += 2.0 * M_PI;
    return angle;
  }
  WP evaluate(double t) const {  // pr:321-331
    WP p;
    p.control = control;
    for (int k = 0; k < dim; k++) {
      p.pos[k] = ax[k].p(t);
      p.vel[k] = ax[k].v(t);
      p.acc[k] = ax[k].a(t);
      p.jrk[k] = ax[k].j(t);
      if (control & USE_YAW) p.yaw = normalize_angle(yawp.p(t));
    }
    return p;
  }
  double max_vel(int k) const {  // pr:353-363
    std::vector<double> ts = ax[k].extrema_v(T);
    double m = std::max(std::abs(ax[k].v(0)), std::abs(ax[k].v(T)));
    for (double it : ts)
      if (it > 0 && it < T) { double v = std::abs(ax[k].v(it)); m = v > m ? v : m; }
    return m;
  }
  double max_acc(int k) const {  // pr:369-379
    std::vector<double> ts = ax[k].extrema_a(T);
    double m = std::max(std::abs(ax[k].a(0)), std::abs(ax[k].a(T)));
    for (double it : ts)
      if (it > 0 && it < T) { double a = std::abs(ax[k].a(it)); m = a > m ? a : m; }
    return m;
  }
  double max_jrk(int k) const {  // pr:384-394
    std::vector<double> ts = ax[k].extrema_j(T);
    double m = std::max(std::abs(ax[k].j(0)), std::abs(ax[k].j(T)));
    for (double it : ts)
      if (it > 0 && it < T) { double j = std::abs(ax[k].j(it)); m = j > m ? j : m; }
    return m;
  }
  double J(int ctl) const {  // pr:403-407
    double j = 0;
    for (int k = 0; k < dim; k++) j += ax[k].J(T, ctl);
    return j;
  }
};

bool validate_xxx(const Prim &pr, double max, int which) {  // pr:483-496
  if (max <= 0) return true;
  for (int i = 0; i < pr.dim; i++) {
    if (which == C_VEL && pr.max_vel(i) > max) return false;
    else if (which == C_ACC && pr.max_acc(i) > max) return false;
    else if (which == C_JRK && pr.max_jrk(i) > max) return false;
  }
  return true;
}

/* cos/sin as the reference calls them (libm), or correctly rounded (see crtrig above) */
void trig(int mode, double x, double *sn, double *cs) {
  if (mode == 0) { *sn = std::sin(x); *cs = std::cos(x); }
  else crtrig::sincos_cr(x, sn, cs);
}

/* v.normalized().dot(Vec2f(cos(yaw), sin(yaw))) with Eigen's normalized() = v / sqrt(squaredNorm) (pr:520, em:125) */
double heading_dot(const double *vel, double yaw, int trig_mode) {
  double z = vel[0] * vel[0] + vel[1] * vel[1];
  double nx = vel[0], ny = vel[1];
  if (z > 0) { double q = std::sqrt(z); nx = vel[0] / q; ny = vel[1] / q; }
  double sn, cs;
  trig(trig_mode, yaw, &sn, &cs);
  return nx * cs + ny * sn;
}

bool validate_yaw(const Prim &pr, double my, int trig_mode) {  // pr:503-525
  if (my <= 0) return true;
  WP ws[2] = {pr.evaluate(0), pr.evaluate(pr.T)};
  double sm, cm;
  trig(trig_mode, my, &sm, &cm);
  for (const WP &w : ws) {
    if (w.vel[0] != 0 || w.vel[1] != 0) {
      double d = heading_dot(w.vel, w.yaw, trig_mode);
      if (d < cm) return false;
    }
  }
  return true;
}

bool validate_primitive(const Prim &pr, double mv, double ma, double mj, double myaw = 0, int trig_mode = 0) {  // pr:449-475
  int cc = pr.control;
  if (cc & USE_YAW) {  // pr:462-472: validate_yaw first, then the bounds of the base control
    if (!validate_yaw(pr, myaw, trig_mode)) return false;
    cc &= 15;
    if (cc == C_VEL) return true;
  }
  if (cc == C_ACC) return validate_xxx(pr, mv, C_VEL);
  else if (cc == C_JRK) return validate_xxx(pr, mv, C_VEL) && validate_xxx(pr, ma, C_ACC);
  else if (cc == C_SNP) return validate_xxx(pr, mv, C_VEL) && validate_xxx(pr, ma, C_ACC) && validate_xxx(pr, mj, C_JRK);
  return true;  // VEL and everything else: pr:473-474
}

/* ------------------------------------------------------------------ MapUtil, mu:20-314 */
struct Map {
  int dim = 3;
  int nd[3] = {1, 1, 1};
  double origin[3] = {0, 0, 0};
  double res = 1;
  std::vector<int8_t> data;

  int index(const int *pn) const {  // mu:33-41
    return dim == 2 ? pn[0] + nd[0] * pn[1] : pn[0] + nd[0] * pn[1] + nd[0] * nd[1] * pn[2];
  }
  bool outside(const int *pn) const {  // mu:51-55
    for (int i = 0; i < dim; i++)
      if (pn[i] < 0 || pn[i] >= nd[i]) return true;
    return false;
  }
  bool occupied(const int *pn) const { return outside(pn) ? false : data[index(pn)] == 100; }  // mu:48,64-69
  bool is_free(const int *pn) const {  // mu:44,57-62
    if (outside(pn)) return false;
    int8_t v = data[index(pn)];
    return v < 100 && v >= 0;
  }
  void float_to_int(const double *pt, int *pn) const {  // mu:103-108
    for (int i = 0; i < dim; i++) pn[i] = (int)std::round((pt[i] - origin[i]) / res - 0.5);
  }
  void free_unknown() {  // mu:259-276
    for (auto &v : data)
      if (v == -1) v = 0;
  }
  /* mu:117-134, the cell list itself (used by MapPlanner::setSearchRegion, map_planner.cpp:50-53) */
  void ray_trace(const double *pt1, const double *pt2, std::vector<std::array<int, 3>> &pns) const {
    double diff[3] = {0, 0, 0}, q = 0;
    for (int i = 0; i < dim; i++) {
      diff[i] = pt2[i] - pt1[i];
      double a = std::abs(diff[i] / res);
      if (i == 0 || a > q) q = a;
    }
    int max_diff = (int)(q / 0.8);
    double s = 1.0 / max_diff;
    double step[3] = {0, 0, 0};
    for (int i = 0; i < dim; i++) step[i] = diff[i] * s;
    int prev[3] = {-1, -1, -1};
    for (int n = 1; n < max_diff; n++) {
      double pt[3] = {0, 0, 0};
      int pn[3] = {0, 0, 0};
      for (int i = 0; i < dim; i++) pt[i] = pt1[i] + step[i] * n;
      float_to_int(pt, pn);
      if (outside(pn)) break;
      bool same = true;
      for (int i = 0; i < dim; i++) same = same && pn[i] == prev[i];
      if (!same) pns.push_back({pn[0], pn[1], pn[2]});
      for (int i = 0; i < dim; i++) prev[i] = pn[i];
    }
  }
  /* mu:117-134; returns true iff some traced cell is occupied (what em:38-42 asks). */
  bool ray_hits_occupied(const double *pt1, const double *pt2) const {
    double diff[3], q = 0;
    for (int i = 0; i < dim; i++) {
      diff[i] = pt2[i] - pt1[i];
      double a = std::abs(diff[i] / res);
      if (i == 0 || a > q) q = a;  // lpNorm<Infinity>
    }
    int max_diff = (int)(q / 0.8);
    double s = 1.0 / max_diff;
    double step[3];
    for (int i = 0; i < dim; i++) step[i] = diff[i] * s;
    for (int n = 1; n < max_diff; n++) {
      double pt[3];
      int pn[3] = {0, 0, 0};
      for (int i = 0; i < dim; i++) pt[i] = pt1[i] + step[i] * n;
      float_to_int(pt, pn);
      if (outside(pn)) break;
      if (data[index(pn)] == 100) return true;
    }
    return false;
  }
};

/* ------------------------------------------------------------------ Boost d_ary_heap<arity<2>, mutable_<true>>
 * Restated from Boost.Heap's published algorithm (boost/heap/d_ary_heap.hpp, stable since 1.49):
 *   push      : append, sift UP while cmp(parent, x)  (parent strictly worse than x)
 *   pop       : swap(front, back), drop back, sift DOWN the new front
 *   sift down : best child = std::max_element over the (<= 2) children w.r.t. cmp (FIRST of equal
 *               maxima, i.e. the left child on ties); swap unless cmp(best child, x) (child strictly
 *               worse than x) — so on a tie the element still moves down
 *   increase  : sift UP from the element's position (gs:133 calls increase after lowering f)
 * cmp = compare_pair (ss:15-27): cmp(a,b) true iff a is WORSE than b:
 *   a.f == b.f ? min(g_a,rhs_a) > min(g_b,rhs_b) : a.f > b.f ; g is read through the node pointer
 *   at comparison time (rhs stays +inf in A*).                                                     */
struct Node {
  WP coord;
  Key key;
  double g = kInf, h = kInf;
  bool opened = false, closed = false;
  int heap_entry = -1;  // handle
  std::vector<int> pred_node;  // gs:100-102 (node ids instead of coords; hm_ lookup is by key either way)
  std::vector<double> pred_cost;
  std::vector<int> pred_act;
};

struct Heap {
  struct Entry { double f; int node; int pos; };
  std::vector<Entry> entries;  // stable storage (the std::list of the mutable heap)
  std::vector<int> q;          // heap order: entry ids
  const std::vector<Node> *nodes = nullptr;

  bool worse(int ea, int eb) const {
    const Entry &a = entries[ea], &b = entries[eb];
    if (a.f == b.f) return (*nodes)[a.node].g > (*nodes)[b.node].g;
    return a.f > b.f;
  }
  void place(int pos, int e) { q[pos] = e; entries[e].pos = pos; }
  void sift_up(int pos) {
    while (pos != 0) {
      int parent = (pos - 1) / 2;
      if (worse(q[parent], q[pos])) {
        int a = q[parent], b = q[pos];
        place(parent, b); place(pos, a);
        pos = parent;
      } else return;
    }
  }
  void sift_down(int pos) {
    int n = (int)q.size();
    while (2 * pos + 1 < n) {
      int c = 2 * pos + 1;
      if (c + 1 < n && worse(q[c], q[c + 1])) c = c + 1;  // max_element: later one only if strictly better
      if (!worse(q[c], q[pos])) {
        int a = q[c], b = q[pos];
        place(pos, a); place(c, b);
        pos = c;
      } else return;
    }
  }
  int push(double f, int node) {
    int e = (int)entries.size();
    entries.push_back({f, node, (int)q.size()});
    q.push_back(e);
    sift_up((int)q.size() - 1);
    return e;
  }
  int top_node() const { return entries[q[0]].node; }
  void pop() {
    int last = q.back();
    q.pop_back();
    if (q.empty()) return;
    place(0, last);
    sift_down(0);
  }
  void increase(int e, double f) { entries[e].f = f; sift_up(entries[e].pos); }
  bool empty() const { return q.empty(); }
};

/* ------------------------------------------------------------------ planner (env_map + env_base + Astar) */
struct Planner {
  int dim = 3;
  Map *map = nullptr;
  // env_base defaults eb:368-392; planner defaults pb:337-339
  double w = 10.0, tol_pos = 0.5, tol_vel = -1.0, tol_acc = -1.0;
  double v_max = -1.0, a_max = -1.0, j_max = -1.0, yaw_max = -1.0, dt = 1.0;
  double eps = 1.0;
  double wyaw = 1.0, tol_yaw = -1.0;  // eb:372,380
  int trig_mode = 0;                  // 0 = libm cos/sin (the reference), 1 = correctly rounded (see crtrig)
  int max_num = -1;
  std::vector<std::vector<double>> U;
  WP goal;
  // cost shaping (em:104-118, eb:395-396; MapPlanner members map_planner.h:104-118)
  std::vector<int8_t> potential_map;
  std::vector<bool> search_region;
  std::vector<std::pair<WP, double>> prior;  // eb:397 prior_traj_
  WP prior_goal;                             // em:224: goal_node_ = traj.evaluate(total_time)
  double potential_weight = 0.1, gradient_weight = 0.0;  // em:294-296
  double search_radius[3] = {0, 0, 0}, potential_radius[3] = {0, 0, 0}, potential_map_range[3] = {0, 0, 0};
  double pow_ = 1.0;
  int8_t H_MAX = 100;

  // state of the last plan
  std::vector<Node> nodes;
  std::unordered_map<Key, int, KeyHasher> hm;
  Heap heap;
  std::vector<int> pop_order;
  std::vector<int> traj_actions;
  std::vector<int> traj_nodes;  // parent node of each segment
  // largest hm_.size(), pq_.size() and predecessor-record count seen when an expansion starts (after its pop, before get_succ):
  // the point where the CUDA kernel checks its arena capacity (orc_get_peaks)
  int64_t peak_nodes = 0, peak_heap = 0, peak_records = 0;
  long long dbg_increase = 0, dbg_pred_total = 0, dbg_pred_hit = 0, dbg_pred_new = 0;
  int dbg_pred = -1, dbg_nodes_before = 0;  // decrease-key events (diagnostics, printed when ORC_DEBUG is set)
  orc_result last;

  /* em:25-45 */
  bool is_goal(const WP &s) const {
    double m = 0;
    for (int i = 0; i < dim; i++) m = std::max(m, std::abs(s.pos[i] - goal.pos[i]));
    bool goaled = m <= tol_pos;
    if (goaled && tol_vel >= 0) {
      m = 0;
      for (int i = 0; i < dim; i++) m = std::max(m, std::abs(s.vel[i] - goal.vel[i]));
      goaled = m <= tol_vel;
    }
    if (goaled && tol_acc >= 0) {
      m = 0;
      for (int i = 0; i < dim; i++) m = std::max(m, std::abs(s.acc[i] - goal.acc[i]));
      goaled = m <= tol_acc;
    }
    if (goaled && tol_yaw >= 0) goaled = std::abs(s.yaw - goal.yaw) <= tol_yaw;  // em:36-37
    if (goaled && map->ray_hits_occupied(s.pos, goal.pos)) return false;
    return goaled;
  }

  /* eb:56-64, heur_ignore_dynamics_ = true (default eb:368) */
  double cal_heur(const WP &s, const WP &target) const {
    double m = 0;
    for (int i = 0; i < dim; i++) m = std::max(m, std::abs(s.pos[i] - target.pos[i]));
    if (v_max > 0) return w * m / v_max;
    return w * m;
  }
  /* eb:46-53: with a prior trajectory the heuristic is the distance to the prior's waypoint at the state's own time plus
   * the prior's remaining time cost */
  double get_heur(const WP &s, const Key &skey) const {
    if (make_key(goal, dim) == skey) return 0;
    size_t id = (size_t)(s.t / dt);
    if (!prior.empty() && id < prior.size()) return cal_heur(s, prior[id].first) + prior[id].second;
    return cal_heur(s, goal);
  }
  /* PlannerBase::setPriorTrajectory -> env_base::set_prior_trajectory (pb:249-252, eb:249-256) from the trajectory of
   * `src`'s last plan; Trajectory::evaluate (trajectory.h:66-86) without a time-scaling lambda */
  void set_prior_from(const Planner &src) {
    prior.clear();
    const int n = (int)src.traj_actions.size();
    std::vector<Prim> segs;
    std::vector<double> taus(1, 0.0);
    for (int i = 0; i < n; i++) {
      segs.emplace_back(src.nodes[src.traj_nodes[i]].coord, src.U[src.traj_actions[i]].data(), src.dt, src.dim);
      taus.push_back(segs.back().T + taus.back());  // trajectory.h:52-57
    }
    const double total = taus.back();
    auto evaluate = [&](double time) {  // trajectory.h:66-86
      double tau = time;
      if (tau < 0) tau = 0;
      if (tau > total) tau = total;
      WP p;
      for (size_t id = 0; id < segs.size(); id++) {
        if ((tau >= taus[id] && tau < taus[id + 1]) || id == segs.size() - 1) {
          tau -= taus[id];
          p.control = segs[id].control;
          for (int j = 0; j < dim; j++) {
            p.pos[j] = segs[id].ax[j].p(tau); p.vel[j] = segs[id].ax[j].v(tau);
            p.acc[j] = segs[id].ax[j].a(tau); p.jrk[j] = segs[id].ax[j].j(tau);
            p.yaw = Prim::normalize_angle(segs[id].yawp.p(tau));
          }
          break;
        }
      }
      return p;
    };
    /* em:187-225 without a potential map: costs[id] = w t, total_cost = traverse_trajectory (0 on a free path) + w total,
     * prior cost = total_cost - costs[id]; then the prior's end point becomes the goal */
    const double total_cost = 0.0 + w * total;
    for (double t = 0; t < total; t += dt) prior.push_back(std::make_pair(evaluate(t), total_cost - w * t));
    prior_goal = evaluate(total);
  }

  /* em:90-132 */
  double traverse(const Prim &pr, orc_prim_trace *tr, int64_t *n_samples) const {
    double max_v = 0;
    for (int i = 0; i < dim; i++)
      if (pr.max_vel(i) > max_v) max_v = pr.max_vel(i);
    int n = std::max(5, (int)std::ceil(max_v * pr.T / map->res));
    double c = 0;
    double dts = pr.T / n;
    int tested = 0;
    if (tr) { tr->n = n; tr->block_idx = -1; }
    for (double t = 0; t < pr.T; t += dts) {
      WP pt = pr.evaluate(t);
      int pn[3] = {0, 0, 0};
      map->float_to_int(pt.pos, pn);
      tested++;
      const bool out = map->outside(pn);
      const int idx = out ? -1 : map->index(pn);
      if (out || (!search_region.empty() && !search_region[idx])) {  // em:104-106
        if (tr) { tr->n_tested = tested; tr->block_idx = idx; }
        *n_samples += tested;
        return kInf;
      }
      if (!potential_map.empty()) {  // em:113-118
        if (potential_map[idx] < 100 && potential_map[idx] > 0) {
          double vn = 0;
          for (int k = 0; k < dim; k++) vn += pt.vel[k] * pt.vel[k];  // Eigen norm(): sqrt of the left-to-right sum of squares
          c += dts * (potential_weight * potential_map[idx] + gradient_weight * std::sqrt(vn));
        } else if (potential_map[idx] >= 100) {
          if (tr) { tr->n_tested = tested; tr->block_idx = idx; }
          *n_samples += tested;
          return kInf;
        }
      } else if (map->data[idx] == 100) {  // em:119-120
        if (tr) { tr->n_tested = tested; tr->block_idx = idx; }
        *n_samples += tested;
        return kInf;
      }
      if (wyaw > 0 && (pt.control & USE_YAW)) {  // em:121-128
        double nrm = std::sqrt(pt.vel[0] * pt.vel[0] + pt.vel[1] * pt.vel[1]);
        if (nrm > 1e-5) {
          double v_value = 1 - heading_dot(pt.vel, pt.yaw, trig_mode);
          c += wyaw * v_value * dts;
        }
      }
    }
    if (tr) tr->n_tested = tested;
    *n_samples += tested;
    return c;
  }

  /* MapPlanner::setSearchRegion, map_planner.cpp:46-95 */
  void set_search_region_path(const std::vector<std::array<double, 3>> &path, bool dense) {
    std::vector<std::array<int, 3>> ps;
    if (!dense) {
      for (size_t i = 1; i < path.size(); i++) {
        map->ray_trace(path[i - 1].data(), path[i].data(), ps);
        int pn[3] = {0, 0, 0};
        map->float_to_int(path[i].data(), pn);
        ps.push_back({pn[0], pn[1], pn[2]});
      }
    } else {
      for (const auto &pt : path) { int pn[3] = {0, 0, 0}; map->float_to_int(pt.data(), pn); ps.push_back({pn[0], pn[1], pn[2]}); }
    }
    int rn[3] = {0, 0, 0};
    for (int i = 0; i < dim; i++) rn[i] = (int)std::ceil(search_radius[i] / map->res);
    size_t ncell = 1;
    for (int i = 0; i < dim; i++) ncell *= (size_t)map->nd[i];
    std::vector<bool> in_region(ncell, false);
    for (const auto &it : ps)
      for (int dx = -rn[0]; dx <= rn[0]; dx++)
        for (int dy = -rn[1]; dy <= rn[1]; dy++)
          for (int dz = (dim == 3 ? -rn[2] : 0); dz <= (dim == 3 ? rn[2] : 0); dz++) {
            int pn[3] = {it[0] + dx, it[1] + dy, it[2] + dz};
            if (map->outside(pn)) continue;
            in_region[map->index(pn)] = true;
          }
    search_region = in_region;
  }

  /* MapPlanner::createMask + updatePotentialMap, map_planner.cpp:286-391.  Rewrites the map itself (setMap(dmap)) and
   * hands the result to the environment as its potential map, exactly like the reference. */
  void update_potential_map(const double *pos) {
    std::vector<std::pair<std::array<int, 3>, int8_t>> mask;
    double res = map->res, h_max = H_MAX;
    int rn = (int)std::ceil(potential_radius[0] / res);
    if (dim == 2) {
      for (int nx = -rn; nx <= rn; nx++)
        for (int ny = -rn; ny <= rn; ny++) {
          if (std::hypot(nx, ny) > rn) continue;
          double h = h_max * std::pow((1 - (double)std::hypot(nx, ny) / rn), pow_);
          if (h > 1e-3) mask.push_back({{nx, ny, 0}, (int8_t)h});
        }
    } else {
      int hn = (int)std::ceil(potential_radius[2] / res);
      for (int nx = -rn; nx <= rn; nx++)
        for (int ny = -rn; ny <= rn; ny++)
          for (int nz = -hn; nz <= hn; nz++) {
            if (std::hypot(nx, ny) > rn) continue;
            double h = h_max * std::pow((1 - (double)std::hypot(nx, ny) / rn) * (1 - (double)std::abs(nz) / hn), pow_);
            if (h > 1e-3) mask.push_back({{nx, ny, nz}, (int8_t)h});
          }
    }
    int c1[3] = {0, 0, 0}, c2[3] = {map->nd[0], map->nd[1], dim == 3 ? map->nd[2] : 1};
    double rnorm = 0;
    for (int i = 0; i < dim; i++) rnorm += potential_map_range[i] * potential_map_range[i];
    if (std::sqrt(rnorm) > 0) {
      double lo[3], hi[3];
      for (int i = 0; i < dim; i++) { lo[i] = pos[i] - potential_map_range[i]; hi[i] = pos[i] + potential_map_range[i]; }
      map->float_to_int(lo, c1);
      map->float_to_int(hi, c2);
      for (int i = 0; i < dim; i++) {
        if (c1[i] < 0) c1[i] = 0; else if (c1[i] >= map->nd[i]) c1[i] = map->nd[i] - 1;
        if (c2[i] < 0) c2[i] = 0; else if (c2[i] >= map->nd[i]) c2[i] = map->nd[i] - 1;
      }
      if (dim == 2) { c1[2] = 0; c2[2] = 1; }
    }
    const std::vector<int8_t> src = map->data;
    std::vector<int8_t> dmap = src;
    for (int x = c1[0]; x < c2[0]; x++)
      for (int y = c1[1]; y < c2[1]; y++)
        for (int z = c1[2]; z < c2[2]; z++) {
          int pn[3] = {x, y, z};
          int idx = map->index(pn);
          if (src[idx] > 0) {
            dmap[idx] = H_MAX;
            for (const auto &it : mask) {
              int q[3] = {x + it.first[0], y + it.first[1], z + it.first[2]};
              if (!map->outside(q)) { int qi = map->index(q); dmap[qi] = std::max(dmap[qi], it.second); }
            }
          }
        }
    map->data = dmap;
    potential_map = dmap;
  }

  /* em:147-172.  Emits rows for every u when `trace` is given; succ lists hold only the entries the
   * reference pushes (self-loops and dyn-rejects produce none). */
  void get_succ(const WP &curr, std::vector<WP> &succ, std::vector<double> &cost, std::vector<int> &act,
                orc_prim_trace *trace, int64_t *n_samples) const {
    succ.clear(); cost.clear(); act.clear();
    Key ck = make_key(curr, dim);
    for (size_t i = 0; i < U.size(); i++) {
      Prim pr(curr, U[i].data(), dt, dim);
      WP tn = pr.evaluate(dt);
      Key tk = make_key(tn, dim);
      orc_prim_trace *tr = trace ? &trace[i] : nullptr;
      if (tr) {
        std::memset(tr, 0, sizeof(*tr));
        tr->block_idx = -1;
        for (int k = 0; k < 3; k++) { tr->succ[k] = tn.pos[k]; tr->succ[3 + k] = tn.vel[k]; tr->succ[6 + k] = tn.acc[k]; tr->succ[9 + k] = tn.jrk[k]; }
        tr->succ[12] = tn.yaw;
        for (int k = 0; k < tk.n; k++) tr->key[k] = tk.v[k];
        tr->key[15] = tk.n;
      }
      if (tk == ck) { if (tr) tr->verdict = 0; continue; }
      if (!validate_primitive(pr, v_max, a_max, j_max, yaw_max, trig_mode)) { if (tr) tr->verdict = 1; continue; }
      tn.t = curr.t + dt;
      succ.push_back(tn);
      bool same = true;
      for (int k = 0; k < dim; k++) same = same && (curr.pos[k] == tn.pos[k]);
      double c = same ? 0 : traverse(pr, tr, n_samples);
      if (!std::isinf(c)) c += pr.J(pr.control) + w * dt;  // eb:343-345
      if (tr) { tr->verdict = std::isinf(c) ? 2 : (same ? 4 : 3); tr->cost = c; }
      cost.push_back(c);
      act.push_back((int)i);
    }
  }

  /* ================================================================== LPA* (SURVEY 8f.3)
   * A literal restatement of GraphSearch::LPAstar (gs:194-365), StateSpace::getSubStateSpace / increaseCost / decreaseCost /
   * updateNode / calculateKey (ss:116-282), MapPlanner::getLinkedNodes / updateBlockedNodes / updateClearedNodes
   * (map_planner.cpp:125-185) and env_map::is_free(Primitive) (em:60-76).  Node objects live in `ln` (a new State is a new
   * entry, like make_shared); hm_ is `lhm` (key -> entry) plus `lorder`, its iteration order, defined as INSERTION order
   * (Boost leaves it unspecified; see oracle/shim/boost/unordered_map.hpp).  Boost.Heap's erase = unconditional sift-up to the
   * root, then pop. */
  struct LNode {
    WP coord;
    Key key;
    std::vector<WP> succ_coord; std::vector<int> succ_act; std::vector<double> succ_cost;
    std::vector<WP> pred_coord; std::vector<int> pred_act; std::vector<double> pred_cost;
    int heap_entry = -1;
    double g = kInf, rhs = kInf, h = kInf;
    bool opened = false, closed = false;
  };
  struct LHeap { /* d_ary_heap<pair<fval, StatePtr>, arity<2>, mutable_<true>, compare_pair> */
    struct Entry { double f; int node; int pos; };
    std::vector<Entry> entries;
    std::vector<int> q;
    const std::vector<LNode> *nodes = nullptr;
    bool worse(int ea, int eb) const { /* compare_pair, ss:15-27 */
      const Entry &a = entries[ea], &b = entries[eb];
      if (a.f == b.f) {
        const LNode &na = (*nodes)[a.node], &nb = (*nodes)[b.node];
        return std::min(na.g, na.rhs) > std::min(nb.g, nb.rhs);
      }
      return a.f > b.f;
    }
    void place(int pos, int e) { q[pos] = e; entries[e].pos = pos; }
    void sift_up(int pos, bool force) {
      while (pos != 0) {
        int parent = (pos - 1) / 2;
        if (force || worse(q[parent], q[pos])) { int a = q[parent], b = q[pos]; place(parent, b); place(pos, a); pos = parent; }
        else return;
      }
    }
    void sift_down(int pos) {
      int n = (int)q.size();
      while (2 * pos + 1 < n) {
        int c = 2 * pos + 1;
        if (c + 1 < n && worse(q[c], q[c + 1])) c = c + 1;
        if (!worse(q[c], q[pos])) { int a = q[c], b = q[pos]; place(pos, a); place(c, b); pos = c; }
        else return;
      }
    }
    int push(double f, int node) {
      int e = (int)entries.size();
      entries.push_back({f, node, (int)q.size()});
      q.push_back(e);
      sift_up((int)q.size() - 1, false);
      return e;
    }
    void pop() {
      int last = q.back();
      int first = q[0];
      place(0, last);
      q.pop_back();
      entries[first].pos = -1;
      if (!q.empty()) sift_down(0);
    }
    void erase(int e) { sift_up(entries[e].pos, true); pop(); }
    bool empty() const { return q.empty(); }
    void clear() { q.clear(); entries.clear(); }
  };
  std::vector<LNode> ln;
  std::unordered_map<Key, int, KeyHasher> lhm;
  std::vector<int> lorder; /* hm_ iteration order */
  LHeap lpq;
  std::vector<int> best_child;
  double l_eps = 1, start_g = 0, start_rhs = 0, start_t = 0;
  bool lpa_init = false;
  int l_expand_iteration = 0;
  std::vector<int> ltraj_actions, ltraj_nodes;
  std::vector<Key> l_explored; /* nodes whose successors were generated in the last call */
  bool lpa_fault = false;      /* a step the reference leaves undefined was reached (see lpa_sub_state_space) */
  bool lpa_cycle = false;      /* the last trace-back ran into a predecessor cycle (the reference would not terminate) */
  /* lhm_ of MapPlanner: voxel index -> (node coord, pred index) in insertion order */
  std::unordered_map<int, std::vector<std::pair<Key, int>>> linked;

  void lpa_reset() { /* pb:164-167 */
    ln.clear(); lhm.clear(); lorder.clear(); lpq.clear(); best_child.clear(); lpa_init = false;
    start_g = start_rhs = start_t = 0; l_expand_iteration = 0; ltraj_actions.clear(); ltraj_nodes.clear(); linked.clear();
  }
  int l_find(const Key &k) const { auto it = lhm.find(k); return it == lhm.end() ? -1 : it->second; }
  int l_new_state(const WP &c) { /* make_shared<State>(coord); h as gs:279-281 */
    LNode n;
    n.coord = c;
    n.key = make_key(c, dim);
    ln.push_back(n);
    return (int)ln.size() - 1;
  }
  double l_key(int id) const { return std::min(ln[id].g, ln[id].rhs) + l_eps * ln[id].h; } /* ss:270-272 */
  void l_update_node(int id) { /* ss:242-267 */
    if (ln[id].rhs != start_rhs) {
      ln[id].rhs = kInf;
      for (size_t i = 0; i < ln[id].pred_coord.size(); i++) {
        const int p = l_find(make_key(ln[id].pred_coord[i], dim));
        if (ln[id].rhs > ln[p].g + ln[id].pred_cost[i]) ln[id].rhs = ln[p].g + ln[id].pred_cost[i];
      }
    }
    if (ln[id].opened && !ln[id].closed) { lpq.erase(ln[id].heap_entry); ln[id].closed = true; }
    if (ln[id].g != ln[id].rhs) {
      ln[id].heap_entry = lpq.push(l_key(id), id);
      ln[id].opened = true;
      ln[id].closed = false;
    }
  }
  /* em:60-76 */
  bool is_free_prim(const Prim &pr) const {
    double max_v = 0;
    for (int i = 0; i < dim; i++)
      if (pr.max_vel(i) > max_v) max_v = pr.max_vel(i);
    const int n = (int)std::ceil(max_v * pr.T / map->res);
    const double dts = pr.T / n; /* Primitive::sample, pr:415-420: N + 1 points at i * dt */
    for (int i = 0; i <= n; i++) {
      WP pt = pr.evaluate(i * dts);
      int pn[3] = {0, 0, 0};
      map->float_to_int(pt.pos, pn);
      if (map->occupied(pn) || map->outside(pn)) return false;
      if (!search_region.empty() && !search_region[map->index(pn)]) return false;
    }
    return true;
  }

  int lpa_plan(const WP &start, const WP &goal_) {
    std::memset(&last, 0, sizeof(last));
    last.cost = kInf;
    l_explored.clear();
    lpa_cycle = false;
    int pn[3] = {0, 0, 0};
    map->float_to_int(start.pos, pn);
    if (!map->is_free(pn)) { last.status = 1; return 1; } /* pb:283-287 */
    if (!lpa_init) { lpa_reset(); lpa_init = true; l_eps = eps; lpq.nodes = &ln; } /* pb:296-304: StateSpace(epsilon_) only once */
    lpq.nodes = &ln;
    goal = goal_; /* pb:306 */
    if (is_goal(start)) { last.status = 5; last.cost = 0; return 5; } /* gs:200-205 */
    const Key skey = make_key(start, dim);
    int curr = l_find(skey); /* gs:208: hm_[start_coord] (inserts the slot) */
    if (curr < 0) {
      curr = l_new_state(start);
      ln[curr].g = kInf;
      ln[curr].rhs = 0;
      ln[curr].h = l_eps == 0 ? 0 : get_heur(start, skey);
      ln[curr].heap_entry = lpq.push(l_key(curr), curr);
      ln[curr].opened = true;
      ln[curr].closed = false;
      lhm[skey] = curr;
      lorder.push_back(curr);
    }
    /* gs:224-241: goal node */
    int goal_node;
    if (!best_child.empty() && is_goal(ln[best_child.back()].coord)) goal_node = best_child.back();
    else {
      goal_node = l_new_state(WP()); /* a detached State(Coord()): never in hm_ */
      ln[goal_node].g = kInf; ln[goal_node].rhs = kInf; ln[goal_node].h = 0;
    }
    int expand_iteration = 0;
    int status = 0;
    std::vector<WP> succ; std::vector<double> scost; std::vector<int> sact;
    while (true) {
      if (lpq.empty()) { status = 3; break; } /* the reference would read pq_.top() of an empty heap here: undefined; reported as "queue empty" */
      if (!(lpq.entries[lpq.q[0]].f < l_key(goal_node) || ln[goal_node].rhs != ln[goal_node].g)) break; /* gs:244-245 */
      expand_iteration++;
      curr = lpq.entries[lpq.q[0]].node;
      lpq.pop();
      ln[curr].closed = true;
      if (ln[curr].g > ln[curr].rhs) ln[curr].g = ln[curr].rhs; /* gs:252-257 */
      else { ln[curr].g = kInf; l_update_node(curr); }
      succ = ln[curr].succ_coord; scost = ln[curr].succ_cost; sact = ln[curr].succ_act; /* gs:261-272 */
      const bool explored = !ln[curr].succ_coord.empty();
      if (!explored) {
        l_explored.push_back(ln[curr].key);
        last.n_prims += (int64_t)U.size();
        WP cw = ln[curr].coord;
        get_succ(cw, succ, scost, sact, nullptr, &last.n_samples);
        for (double c : scost) if (!std::isinf(c)) last.n_valid++;
        ln[curr].succ_coord.resize(succ.size()); ln[curr].succ_act.resize(succ.size()); ln[curr].succ_cost.resize(succ.size());
      }
      for (size_t s = 0; s < succ.size(); s++) { /* gs:287-316 */
        const Key sk = make_key(succ[s], dim);
        int sid = l_find(sk);
        if (sid < 0) {
          sid = l_new_state(succ[s]);
          ln[sid].h = l_eps == 0 ? 0 : get_heur(succ[s], sk);
          lhm[sk] = sid;
          lorder.push_back(sid);
        }
        ln[curr].succ_coord[s] = succ[s]; ln[curr].succ_act[s] = sact[s]; ln[curr].succ_cost[s] = scost[s];
        int id = -1;
        for (size_t i = 0; i < ln[sid].pred_coord.size(); i++)
          if (make_key(ln[sid].pred_coord[i], dim) == ln[curr].key) { id = (int)i; break; }
        if (id == -1) {
          ln[sid].pred_coord.push_back(ln[curr].coord);
          ln[sid].pred_cost.push_back(scost[s]);
          ln[sid].pred_act.push_back(sact[s]);
        }
        l_update_node(sid);
      }
      if (is_goal(ln[curr].coord)) goal_node = curr;                                    /* gs:319 */
      if (max_num > 0 && expand_iteration >= max_num) { status = 2; break; }            /* gs:322-328 */
      if (lpq.empty()) { status = 3; break; }                                           /* gs:331-336 */
    }
    auto fill = [&]() {
      last.n_nodes = (int)lorder.size();
      last.n_open = (int)lpq.q.size();
      uint64_t ch = 0; int nc = 0;
      for (int id : lorder) if (ln[id].closed) { ch += key_hash(ln[id].key); nc++; }
      last.n_closed = nc; last.closed_hash = ch;
      uint64_t ph = 0xCBF29CE484222325ull;
      for (const Key &k : l_explored) ph = (ph ^ key_hash(k)) * 0x100000001B3ull;
      last.pop_hash = ph;
    };
    if (status != 0) { last.status = status; last.pops = expand_iteration; fill(); return status; }
    l_expand_iteration = expand_iteration; /* gs:358 */
    last.pops = expand_iteration;
    /* recoverTraj, gs:369-455 (best_child_ rebuilt, traj_ replaced even on failure) */
    best_child.clear();
    ltraj_actions.clear(); ltraj_nodes.clear();
    bool found = false;
    int c = goal_node;
    std::vector<int> acts, parents;
    while (!ln[c].pred_coord.empty()) {
      if (best_child.size() > lorder.size()) { /* more steps than hm_ has members: a cycle of best predecessors.  The reference's loop
                                                  (gs:377-438) would never return; here the trace-back fails and best_child_ is left empty */
        lpa_cycle = true;
        break;
      }
      best_child.push_back(c);
      int min_id = -1;
      double min_rhs = kInf, min_g = kInf;
      const LNode &cn = ln[c];
      for (size_t i = 0; i < cn.pred_coord.size(); i++) {
        const double pg = ln[l_find(make_key(cn.pred_coord[i], dim))].g;
        if (min_rhs > pg + cn.pred_cost[i]) { min_rhs = pg + cn.pred_cost[i]; min_g = pg; min_id = (int)i; }
        else if (!std::isinf(cn.pred_cost[i]) && min_rhs == pg + cn.pred_cost[i]) {
          if (min_g < pg) { min_g = pg; min_id = (int)i; }
        }
      }
      if (min_id >= 0) {
        acts.push_back(cn.pred_act[min_id]);
        c = l_find(make_key(cn.pred_coord[min_id], dim));
        parents.push_back(c);
      } else break;
      if (ln[c].key == skey) { best_child.push_back(c); found = true; break; }
    }
    std::reverse(best_child.begin(), best_child.end());
    if (lpa_cycle) { best_child.clear(); found = false; }
    fill();
    if (!found) { last.status = 4; return 4; }
    std::reverse(acts.begin(), acts.end());
    std::reverse(parents.begin(), parents.end());
    ltraj_actions = acts; ltraj_nodes = parents;
    last.n_seg = (int)acts.size();
    last.cost = ln[goal_node].g - start_g; /* gs:362 */
    last.status = 0;
    return 0;
  }

  /* ss:116-204 */
  int lpa_sub_state_space(int time_step) {
    if (best_child.empty() || time_step < 0 || time_step >= (int)best_child.size()) return (int)lorder.size();
    int curr = best_child[time_step];
    start_g = ln[curr].g; start_rhs = ln[curr].rhs; start_t = ln[curr].coord.t;
    ln[curr].pred_cost.clear(); ln[curr].pred_act.clear(); ln[curr].pred_coord.clear();
    for (int id : lorder) {
      ln[id].g = kInf; ln[id].rhs = kInf;
      ln[id].pred_cost.clear(); ln[id].pred_act.clear(); ln[id].pred_coord.clear();
    }
    ln[curr].g = start_g; ln[curr].rhs = start_rhs;
    std::unordered_map<Key, int, KeyHasher> new_hm;
    std::vector<int> new_order;
    LHeap epq;
    epq.nodes = &ln;
    ln[curr].heap_entry = epq.push(ln[curr].rhs, curr);
    new_hm[ln[curr].key] = curr; new_order.push_back(curr);
    while (!epq.empty()) {
      curr = epq.entries[epq.q[0]].node;
      epq.pop();
      for (size_t i = 0; i < ln[curr].succ_coord.size(); i++) {
        const Key sk = make_key(ln[curr].succ_coord[i], dim);
        int sid;
        auto it = new_hm.find(sk);
        if (it == new_hm.end()) { /* ss:158-159 */
          sid = l_find(sk);
          if (sid < 0) { lpa_fault = true; continue; } /* "critical bug!!!!" (ss:160-163): the reference dereferences a null State here */
          new_hm[sk] = sid; new_order.push_back(sid);
        } else sid = it->second;
        int id = -1;
        for (size_t k = 0; k < ln[sid].pred_coord.size(); k++)
          if (make_key(ln[sid].pred_coord[k], dim) == ln[curr].key) { id = (int)k; break; }
        if (id == -1) {
          ln[sid].pred_coord.push_back(ln[curr].coord);
          ln[sid].pred_cost.push_back(ln[curr].succ_cost[i]);
          ln[sid].pred_act.push_back(ln[curr].succ_act[i]);
        }
        const double tentative = ln[curr].rhs + ln[curr].succ_cost[i];
        if (tentative < ln[sid].rhs) {
          ln[sid].rhs = tentative;
          if (ln[sid].closed) {
            ln[sid].g = ln[sid].rhs;
            ln[sid].heap_entry = epq.push(ln[sid].rhs, sid);
          }
        }
      }
    }
    lhm = new_hm; lorder = new_order;
    lpq.clear();
    lpq.nodes = &ln;
    for (int id : lorder)
      if (ln[id].opened && !ln[id].closed) ln[id].heap_entry = lpq.push(l_key(id), id);
    return (int)lorder.size();
  }

  /* map_planner.cpp:125-158 */
  int lpa_linked_nodes(std::vector<std::array<double, 3>> &pts) {
    linked.clear();
    pts.clear();
    for (int nid : lorder) {
      const LNode &nd_ = ln[nid];
      for (size_t i = 0; i < nd_.pred_coord.size(); i++) {
        const int p = l_find(make_key(nd_.pred_coord[i], dim));
        Prim pr(ln[p].coord, U[nd_.pred_act[i]].data(), dt, dim);
        double max_v = 0;
        for (int k = 0; k < dim; k++) max_v = std::max(max_v, pr.max_vel(k));
        const int n = (int)(1.0 * std::ceil(max_v * pr.T / map->res));
        int prev_id = -1;
        const double dts = pr.T / n;
        for (int s = 0; s <= n; s++) {
          WP w = pr.evaluate(s * dts);
          int pn[3] = {0, 0, 0};
          map->float_to_int(w.pos, pn);
          const int id = map->index(pn);
          if (id != prev_id) {
            std::array<double, 3> q = {0, 0, 0};
            for (int k = 0; k < dim; k++) q[k] = (pn[k] + 0.5) * map->res + map->origin[k]; /* intToFloat, mu:110-114 */
            pts.push_back(q);
            linked[id].push_back(std::make_pair(nd_.key, (int)i));
            prev_id = id;
          }
        }
      }
    }
    return (int)pts.size();
  }
  /* map_planner.cpp:160-185 + ss:207-240 */
  int lpa_update(const int32_t *pns3, int n, bool blocked) {
    std::vector<std::pair<Key, int>> affected;
    for (int i = 0; i < n; i++) {
      int pn[3] = {pns3[i * 3], pns3[i * 3 + 1], pns3[i * 3 + 2]};
      const int id = map->index(pn);
      auto it = linked.find(id);
      if (it != linked.end()) for (const auto &nd_ : it->second) affected.push_back(nd_);
    }
    for (const auto &a : affected) {
      const int sid = l_find(a.first);
      const int i = a.second;
      if (blocked) { /* increaseCost */
        if (!std::isinf(ln[sid].pred_cost[i])) {
          ln[sid].pred_cost[i] = kInf;
          l_update_node(sid);
          const int p = l_find(make_key(ln[sid].pred_coord[i], dim));
          const int act = ln[sid].pred_act[i];
          for (size_t j = 0; j < ln[p].succ_act.size(); j++)
            if (act == ln[p].succ_act[j]) { ln[p].succ_cost[j] = kInf; break; }
        }
      } else { /* decreaseCost */
        if (std::isinf(ln[sid].pred_cost[i])) {
          const WP parent_key = ln[sid].pred_coord[i];
          Prim pr(parent_key, U[ln[sid].pred_act[i]].data(), dt, dim);
          if (is_free_prim(pr)) {
            ln[sid].pred_cost[i] = pr.J(pr.control) + w * dt; /* eb:343-345 */
            l_update_node(sid);
            const int p = l_find(make_key(parent_key, dim));
            const int act = ln[sid].pred_act[i];
            for (size_t j = 0; j < ln[p].succ_act.size(); j++)
              if (act == ln[p].succ_act[j]) { ln[p].succ_cost[j] = ln[sid].pred_cost[i]; break; }
          }
        }
      }
    }
    return (int)affected.size();
  }

  int plan(const WP &start, const WP &goal_) {
    nodes.clear(); hm.clear(); heap = Heap(); pop_order.clear(); traj_actions.clear(); traj_nodes.clear();
    peak_nodes = peak_heap = peak_records = 0;
    std::memset(&last, 0, sizeof(last));
    last.cost = kInf;
    heap.nodes = &nodes;
    // pb:283-287
    int pn[3] = {0, 0, 0};
    map->float_to_int(start.pos, pn);
    if (!map->is_free(pn)) { last.status = 1; return 1; }
    if (prior.empty()) goal = goal_;  // eb:295-298: with a prior trajectory the requested goal is ignored ...
    else goal = prior_goal;          // ... and the goal stays the prior's end point (em:224)
    // gs:44
    if (is_goal(start)) { last.status = 5; last.cost = 0; return 5; }
    // gs:47-60
    {
      Node n0;
      n0.coord = start;
      n0.key = make_key(start, dim);
      n0.g = 0;
      n0.h = eps == 0 ? 0 : get_heur(start, n0.key);
      n0.opened = true;
      nodes.push_back(n0);
      hm[n0.key] = 0;
      nodes[0].heap_entry = heap.push(nodes[0].g + eps * nodes[0].h, 0);
    }
    int expand_iteration = 0;
    int curr = -1;
    std::vector<WP> succ; std::vector<double> scost; std::vector<int> sact;
    uint64_t pop_hash = 0xCBF29CE484222325ull, closed_hash = 0;
    int n_closed = 0;
    int status = 0;
    while (true) {
      expand_iteration++;
      curr = heap.top_node();
      if (dbg_pred >= 0) { dbg_pred_total++; if (dbg_pred == curr) dbg_pred_hit++; else if (curr >= dbg_nodes_before) dbg_pred_new++; }
      heap.pop();
      dbg_pred = heap.empty() ? -1 : heap.top_node();
      dbg_nodes_before = (int)nodes.size();
      peak_nodes = std::max<int64_t>(peak_nodes, (int64_t)nodes.size());
      peak_heap = std::max<int64_t>(peak_heap, (int64_t)heap.q.size());
      peak_records = std::max<int64_t>(peak_records, last.n_valid); /* one record per finite-cost edge so far (gs:100-102) */
      uint64_t kh = key_hash(nodes[curr].key);
      pop_hash = (pop_hash ^ kh) * 0x100000001B3ull;
      if (!nodes[curr].closed) { n_closed++; closed_hash += kh; }
      nodes[curr].closed = true;
      pop_order.push_back(curr);
      last.n_prims += (int64_t)U.size();
      WP cw = nodes[curr].coord;
      get_succ(cw, succ, scost, sact, nullptr, &last.n_samples);
      for (size_t s = 0; s < succ.size(); s++) {
        if (std::isinf(scost[s])) continue;  // gs:81
        last.n_valid++;
        Key sk = make_key(succ[s], dim);
        auto it = hm.find(sk);
        int sid;
        if (it == hm.end()) {  // gs:84-88
          sid = (int)nodes.size();
          Node nn;
          nn.coord = succ[s];
          nn.key = sk;
          nn.h = eps == 0 ? 0 : get_heur(succ[s], sk);
          nodes.push_back(nn);
          hm[sk] = sid;
        } else sid = it->second;
        Node &sn = nodes[sid];
        sn.pred_node.push_back(curr);  // gs:100-102
        sn.pred_cost.push_back(scost[s]);
        sn.pred_act.push_back(sact[s]);
        double tentative = nodes[curr].g + scost[s];
        if (tentative < sn.g) {  // gs:107-141
          sn.g = tentative;
          double fval = sn.g + eps * sn.h;
          if (sn.opened && !sn.closed) { heap.increase(sn.heap_entry, fval); dbg_increase++; }
          else { sn.heap_entry = heap.push(fval, sid); nodes[sid].opened = true; }
        }
      }
      if (is_goal(nodes[curr].coord)) break;                                             // gs:146
      if (max_num > 0 && expand_iteration >= max_num) { status = 2; break; }             // gs:149-154
      if (heap.empty()) { status = 3; break; }                                           // gs:157-161
    }
    last.pops = expand_iteration;
    if (std::getenv("ORC_DEBUG")) std::fprintf(stderr, "orc: pops %d nodes %zu increase %lld valid %lld pred_hit %.3f pred_new %.3f\n", expand_iteration, nodes.size(), dbg_increase, (long long)last.n_valid, dbg_pred_total ? (double)dbg_pred_hit / dbg_pred_total : 0.0, dbg_pred_total ? (double)dbg_pred_new / dbg_pred_total : 0.0);
    last.n_nodes = (int)nodes.size();
    last.n_open = (int)heap.q.size();
    last.n_closed = n_closed;
    last.pop_hash = pop_hash;
    last.closed_hash = closed_hash;
    if (status != 0) { last.status = status; return status; }
    // recoverTraj gs:369-455
    bool found = false;
    int c = curr;
    std::vector<int> acts, parents;
    while (!nodes[c].pred_node.empty()) {
      int min_id = -1;
      double min_rhs = kInf, min_g = kInf;
      const Node &cn = nodes[c];
      for (size_t i = 0; i < cn.pred_node.size(); i++) {
        double pg = nodes[cn.pred_node[i]].g;
        if (min_rhs > pg + cn.pred_cost[i]) { min_rhs = pg + cn.pred_cost[i]; min_g = pg; min_id = (int)i; }
        else if (!std::isinf(cn.pred_cost[i]) && min_rhs == pg + cn.pred_cost[i]) {
          if (min_g < pg) { min_g = pg; min_id = (int)i; }
        }
      }
      if (min_id >= 0) {
        acts.push_back(cn.pred_act[min_id]);
        c = cn.pred_node[min_id];
        parents.push_back(c);
      } else break;
      if (nodes[c].key == nodes[0].key) { found = true; break; }  // gs:433 (start_key, hash equality)
    }
    if (!found) { last.status = 4; return 4; }
    std::reverse(acts.begin(), acts.end());
    std::reverse(parents.begin(), parents.end());
    traj_actions = acts;
    traj_nodes = parents;
    last.n_seg = (int)acts.size();
    last.cost = nodes[curr].g;  // gs:179
    last.status = 0;
    return 0;
  }
};

}  // namespace

/* ================================================================== C interface */
extern "C" {

void *orc_map_create(int dim, const int32_t *ndim, const double *origin, double res, const int8_t *data) {
  Map *m = new Map();
  m->dim = dim;
  size_t n = 1;
  for (int i = 0; i < dim; i++) { m->nd[i] = ndim[i]; m->origin[i] = origin[i]; n *= (size_t)ndim[i]; }
  m->res = res;
  m->data.assign(data, data + n);  // mu:84-90 deep copy
  return m;
}
void orc_map_destroy(void *map) { delete (Map *)map; }
void orc_map_free_unknown(void *map) { ((Map *)map)->free_unknown(); }
int orc_map_float_to_int(void *map, const double *pt, int32_t *pn) {
  Map *m = (Map *)map;
  int p[3] = {0, 0, 0};
  m->float_to_int(pt, p);
  for (int i = 0; i < m->dim; i++) pn[i] = p[i];
  return m->outside(p) ? -1 : m->index(p);
}

void *orc_planner_create(int dim) { Planner *p = new Planner(); p->dim = dim; return p; }
void orc_planner_destroy(void *p) { delete (Planner *)p; }
void orc_planner_set_map(void *p, void *map) { ((Planner *)p)->map = (Map *)map; }
int orc_planner_set_param(void *pp, const char *key, double v) {
  Planner *p = (Planner *)pp;
  std::string k(key);
  if (k == "v_max") p->v_max = v; else if (k == "a_max") p->a_max = v; else if (k == "j_max") p->j_max = v;
  else if (k == "yaw_max") p->yaw_max = v; else if (k == "dt") p->dt = v; else if (k == "w") p->w = v;
  else if (k == "epsilon") p->eps = v; else if (k == "max_num") p->max_num = (int)v;
  else if (k == "tol_pos") p->tol_pos = v; else if (k == "tol_vel") p->tol_vel = v; else if (k == "tol_acc") p->tol_acc = v;
  else if (k == "potential_weight") p->potential_weight = v; else if (k == "gradient_weight") p->gradient_weight = v;
  else if (k == "pow") p->pow_ = v;
  else if (k == "wyaw") p->wyaw = v; else if (k == "tol_yaw") p->tol_yaw = v; else if (k == "trig_mode") p->trig_mode = (int)v;
  else return -1;
  return 0;
}
void orc_planner_set_controls(void *pp, const double *U, int n, int udim) {
  Planner *p = (Planner *)pp;
  p->U.clear();
  for (int i = 0; i < n; i++) p->U.emplace_back(U + (size_t)i * udim, U + (size_t)(i + 1) * udim);
}

void orc_planner_set_vec(void *pp, const char *key, const double *v) {
  Planner *p = (Planner *)pp;
  std::string k(key);
  double *dst = k == "search_radius" ? p->search_radius : k == "potential_radius" ? p->potential_radius : p->potential_map_range;
  for (int i = 0; i < p->dim; i++) dst[i] = v[i];
}
void orc_planner_set_search_region(void *pp, const double *path, int n, int dense) {
  Planner *p = (Planner *)pp;
  std::vector<std::array<double, 3>> pts(n);
  for (int i = 0; i < n; i++) { pts[i] = {0, 0, 0}; for (int k = 0; k < p->dim; k++) pts[i][k] = path[(size_t)i * 3 + k]; }
  p->set_search_region_path(pts, dense != 0);
}
void orc_planner_set_potential_map(void *pp, const int8_t *pot, int64_t n) { /* env_map::set_potential_map, em:182 */
  Planner *p = (Planner *)pp;
  p->potential_map.assign(pot, pot + (pot ? n : 0));
}
void orc_planner_set_search_region_mask(void *pp, const uint8_t *mask, int64_t n) { /* env_base::set_search_region, eb:301-303 */
  Planner *p = (Planner *)pp;
  p->search_region.assign((size_t)(mask ? n : 0), false);
  for (int64_t i = 0; mask && i < n; i++) p->search_region[i] = mask[i] != 0;
}
void orc_planner_set_prior_trajectory(void *pp, void *src) { /* src = planner whose last plan supplies the trajectory; NULL clears */
  Planner *p = (Planner *)pp;
  if (src) p->set_prior_from(*(Planner *)src); else p->prior.clear();
}
void orc_planner_clear_shaping(void *pp) { Planner *p = (Planner *)pp; p->search_region.clear(); p->potential_map.clear(); }
int64_t orc_planner_get_search_region(void *pp, uint8_t *out, int64_t cap) {
  Planner *p = (Planner *)pp;
  int64_t n = (int64_t)p->search_region.size();
  for (int64_t i = 0; i < n && i < cap; i++) out[i] = p->search_region[i] ? 1 : 0;
  return n;
}
void orc_planner_update_potential_map(void *pp, const double *pos) { ((Planner *)pp)->update_potential_map(pos); }
void orc_sincos_cr(const double *x, int n, double *s, double *c) {
  for (int i = 0; i < n; i++) crtrig::sincos_cr(x[i], &s[i], &c[i]);
}
int64_t orc_map_get_data(void *map, int8_t *out, int64_t cap) {
  Map *m = (Map *)map;
  int64_t n = (int64_t)m->data.size();
  for (int64_t i = 0; i < n && i < cap; i++) out[i] = m->data[i];
  return n;
}

void orc_map_set_cells(void *map, const int32_t *cells3, int n, int8_t value) {
  Map *m = (Map *)map;
  for (int i = 0; i < n; i++) { int pn[3] = {cells3[i * 3], cells3[i * 3 + 1], cells3[i * 3 + 2]}; m->data[m->index(pn)] = value; }
}
void orc_lpa_reset(void *pp) { ((Planner *)pp)->lpa_reset(); }
int orc_lpa_plan(void *pp, const orc_waypoint *start, const orc_waypoint *goal, orc_result *out) {
  Planner *p = (Planner *)pp;
  int st = p->lpa_plan(from_c(*start), from_c(*goal));
  if (out) *out = p->last;
  return st;
}
int orc_lpa_get_sub_state_space(void *pp, int k) { Planner *p = (Planner *)pp; int n = p->lpa_sub_state_space(k); return p->lpa_fault ? -1 : n; }
int orc_lpa_get_linked_nodes(void *pp, double *pts3, int cap) {
  std::vector<std::array<double, 3>> pts;
  const int n = ((Planner *)pp)->lpa_linked_nodes(pts);
  for (int i = 0; i < n && i < cap; i++) for (int k = 0; k < 3; k++) pts3[(size_t)i * 3 + k] = pts[i][k];
  return n;
}
int orc_lpa_update_blocked_nodes(void *pp, const int32_t *pns3, int n) { return ((Planner *)pp)->lpa_update(pns3, n, true); }
int orc_lpa_update_cleared_nodes(void *pp, const int32_t *pns3, int n) { return ((Planner *)pp)->lpa_update(pns3, n, false); }
static uint64_t lpa_mix(uint64_t h, uint64_t x) { return (h ^ x) * 0x100000001B3ull; }
static uint64_t lpa_bits(double d) { uint64_t u; std::memcpy(&u, &d, 8); return u; }
int orc_lpa_dump_nodes(void *pp, orc_lpa_node *nodes, int cap) {
  Planner *p = (Planner *)pp;
  int n = 0;
  for (int id : p->lorder) {
    if (n < cap) {
      orc_lpa_node &o = nodes[n];
      std::memset(&o, 0, sizeof(o));
      const Planner::LNode &st = p->ln[id];
      for (int k = 0; k < st.key.n; k++) o.key[k] = st.key.v[k];
      o.key[15] = st.key.n;
      o.g = st.g; o.rhs = st.rhs; o.h = st.h; o.opened = st.opened; o.closed = st.closed;
      o.n_succ = (int)st.succ_coord.size(); o.n_pred = (int)st.pred_coord.size();
      uint64_t hs = 0xCBF29CE484222325ull, hp = hs;
      for (size_t i = 0; i < st.succ_coord.size(); i++) hs = lpa_mix(lpa_mix(lpa_mix(hs, key_hash(make_key(st.succ_coord[i], p->dim))), (uint64_t)st.succ_act[i]), lpa_bits(st.succ_cost[i]));
      for (size_t i = 0; i < st.pred_coord.size(); i++) hp = lpa_mix(lpa_mix(lpa_mix(hp, key_hash(make_key(st.pred_coord[i], p->dim))), (uint64_t)st.pred_act[i]), lpa_bits(st.pred_cost[i]));
      o.succ_hash = hs; o.pred_hash = hp;
    }
    n++;
  }
  return n;
}
int orc_lpa_dump_heap(void *pp, orc_lpa_heap_entry *e, int cap) {
  Planner *p = (Planner *)pp;
  int n = 0;
  for (int ent : p->lpq.q) {
    if (n < cap) { e[n].fval = p->lpq.entries[ent].f; e[n].key_hash = key_hash(p->ln[p->lpq.entries[ent].node].key); }
    n++;
  }
  return n;
}
int orc_lpa_best_child(void *pp, int32_t *keys16, int cap) {
  Planner *p = (Planner *)pp;
  for (int i = 0; i < (int)p->best_child.size() && i < cap; i++) {
    int32_t *k = keys16 + (size_t)i * 16;
    std::memset(k, 0, 64);
    const Key &key = p->ln[p->best_child[i]].key;
    for (int j = 0; j < key.n; j++) k[j] = key.v[j];
    k[15] = key.n;
  }
  return (int)p->best_child.size();
}
int orc_lpa_best_child_states(void *pp, double *states13, int cap) {
  Planner *p = (Planner *)pp;
  for (int i = 0; i < (int)p->best_child.size() && i < cap; i++) {
    const WP &w = p->ln[p->best_child[i]].coord;
    double *s = states13 + (size_t)i * 13;
    for (int k = 0; k < 3; k++) { s[k] = w.pos[k]; s[3 + k] = w.vel[k]; s[6 + k] = w.acc[k]; s[9 + k] = w.jrk[k]; }
    s[12] = w.yaw;
  }
  return (int)p->best_child.size();
}
int orc_lpa_last_fault(void *pp) { Planner *p = (Planner *)pp; return (p->lpa_fault ? 1 : 0) | (p->lpa_cycle ? 2 : 0); }
int orc_lpa_get_actions(void *pp, int32_t *actions, int cap) {
  Planner *p = (Planner *)pp;
  for (int i = 0; i < (int)p->ltraj_actions.size() && i < cap; i++) actions[i] = p->ltraj_actions[i];
  return (int)p->ltraj_actions.size();
}

int orc_plan(void *pp, const orc_waypoint *start, const orc_waypoint *goal, orc_result *out) {
  Planner *p = (Planner *)pp;
  int st = p->plan(from_c(*start), from_c(*goal));
  if (out) *out = p->last;
  return st;
}
int orc_get_actions(void *pp, int32_t *actions, int cap) {
  Planner *p = (Planner *)pp;
  int n = (int)p->traj_actions.size();
  for (int i = 0; i < n && i < cap; i++) actions[i] = p->traj_actions[i];
  return n;
}
static void pack_state(const WP &w, double *s) {
  for (int k = 0; k < 3; k++) { s[k] = w.pos[k]; s[3 + k] = w.vel[k]; s[6 + k] = w.acc[k]; s[9 + k] = w.jrk[k]; }
  s[12] = w.yaw;
}
int orc_get_seg_states(void *pp, double *states13, int cap) {
  Planner *p = (Planner *)pp;
  int n = (int)p->traj_nodes.size();
  for (int i = 0; i < n && i < cap; i++) pack_state(p->nodes[p->traj_nodes[i]].coord, states13 + 13 * (size_t)i);
  return n;
}
int orc_get_nodes(void *pp, orc_node *out, int cap) {
  Planner *p = (Planner *)pp;
  int n = (int)p->nodes.size();
  for (int i = 0; i < n && i < cap; i++) {
    const Node &nd = p->nodes[i];
    std::memset(&out[i], 0, sizeof(orc_node));
    pack_state(nd.coord, out[i].state);
    out[i].t = nd.coord.t; out[i].g = nd.g; out[i].h = nd.h;
    for (int k = 0; k < nd.key.n; k++) out[i].key[k] = nd.key.v[k];
    out[i].key[15] = nd.key.n;
    out[i].opened = nd.opened; out[i].closed = nd.closed;
  }
  return n;
}
int orc_get_heap(void *pp, orc_heap_entry *out, int cap) {
  Planner *p = (Planner *)pp;
  int n = (int)p->heap.q.size();
  for (int i = 0; i < n && i < cap; i++) {
    const Heap::Entry &e = p->heap.entries[p->heap.q[i]];
    const Key &k = p->nodes[e.node].key;
    std::memset(&out[i], 0, sizeof(orc_heap_entry));
    for (int j = 0; j < k.n; j++) out[i].key[j] = k.v[j];
    out[i].key[15] = k.n;
    out[i].f = e.f;
    out[i].key_hash = key_hash(k);
  }
  return n;
}
void orc_get_peaks(void *pp, int64_t *peaks3) {
  Planner *p = (Planner *)pp;
  peaks3[0] = p->peak_nodes; peaks3[1] = p->peak_heap; peaks3[2] = p->peak_records;
}
int orc_get_pop_keys(void *pp, int32_t *keys16, int cap) {
  Planner *p = (Planner *)pp;
  int n = (int)p->pop_order.size();
  for (int i = 0; i < n && i < cap; i++) {
    const Key &k = p->nodes[p->pop_order[i]].key;
    int32_t *row = keys16 + 16 * (size_t)i;
    std::memset(row, 0, 16 * sizeof(int32_t));
    for (int j = 0; j < k.n; j++) row[j] = k.v[j];
    row[15] = k.n;
  }
  return n;
}
int orc_get_succ_trace(void *pp, const orc_waypoint *curr, orc_prim_trace *rows, int cap) {
  Planner *p = (Planner *)pp;
  int n = (int)p->U.size();
  if (cap < n) return n;
  std::vector<WP> succ; std::vector<double> c; std::vector<int> a;
  int64_t ns = 0;
  p->get_succ(from_c(*curr), succ, c, a, rows, &ns);
  return n;
}

/* Dynamic work queue: threads pull the next plan index from an atomic counter (in `order` when given, e.g. longest
 * first), one private planner per thread (the reference is single-threaded per plan), threads optionally pinned to
 * cores tid % ncores.  busy_s (nthreads doubles, may be NULL) receives each thread's time inside plan(). */
int orc_plan_batch_dyn(void *pp, const orc_waypoint *starts, const orc_waypoint *goals, int n, int nthreads,
                       orc_result *results, int32_t *actions, int max_seg, const int32_t *order, int pin, double *busy_s) {
  Planner *base = (Planner *)pp;
  if (nthreads < 1) nthreads = 1;
  std::atomic<int> next{0};
  auto worker = [&](int tid) {
    if (pin) {
      cpu_set_t set;
      CPU_ZERO(&set);
      long nc = sysconf(_SC_NPROCESSORS_ONLN);
      CPU_SET((int)(tid % (nc > 0 ? nc : 1)), &set);
      pthread_setaffinity_np(pthread_self(), sizeof(set), &set);
    }
    Planner local;  // same parameters, private search state
    local.dim = base->dim; local.map = base->map; local.w = base->w; local.tol_pos = base->tol_pos;
    local.tol_vel = base->tol_vel; local.tol_acc = base->tol_acc; local.v_max = base->v_max; local.a_max = base->a_max;
    local.j_max = base->j_max; local.yaw_max = base->yaw_max; local.dt = base->dt; local.eps = base->eps;
    local.max_num = base->max_num; local.U = base->U;
    local.potential_map = base->potential_map; local.search_region = base->search_region;
    local.potential_weight = base->potential_weight; local.gradient_weight = base->gradient_weight;
    local.wyaw = base->wyaw; local.tol_yaw = base->tol_yaw; local.trig_mode = base->trig_mode;
    local.prior = base->prior; local.prior_goal = base->prior_goal;
    double busy = 0.0;
    while (true) {
      const int q = next.fetch_add(1);
      if (q >= n) break;
      const int i = order ? order[q] : q;
      auto t0 = std::chrono::steady_clock::now();
      local.plan(from_c(starts[i]), from_c(goals[i]));
      const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      busy += el;
      results[i] = local.last;
      results[i].device_ms = el * 1e3;
      if (actions) {
        int ns = (int)local.traj_actions.size();
        for (int k = 0; k < max_seg; k++) actions[(size_t)i * max_seg + k] = k < ns ? local.traj_actions[k] : -1;
      }
    }
    if (busy_s) busy_s[tid] = busy;
  };
  std::vector<std::thread> th;
  for (int t = 0; t < nthreads; t++) th.emplace_back(worker, t);
  for (auto &t : th) t.join();
  return 0;
}

int orc_plan_batch(void *pp, const orc_waypoint *starts, const orc_waypoint *goals, int n, int nthreads,
                   orc_result *results, int32_t *actions, int max_seg) {
  return orc_plan_batch_dyn(pp, starts, goals, n, nthreads, results, actions, max_seg, nullptr, 0, nullptr);
}

}  // extern "C"
