/*
 * mplb_ref.h — the reference's primitive and map arithmetic, restated once, literally, for host and device.
 *
 * What it restates (paths under motion_primitive_library/include/):
 *   math.h (mt)          normalize_angle :15-19, quad / solve :22-33,117-131, power :197-203
 *   primitive.h (pr)     Primitive1D p/v/a/j :128-145, J :92-122, extrema :152-193; Primitive from (state, u, control order)
 *                        :35-52,220-256, evaluate :321-331, max_vel / max_acc / max_jrk :353-394, validatePrimitive :449-496
 *   map_util.h (mu)      cell index :33-41, outside :51-55, floatToInt :103-108, rayTrace step rule :117-134
 * and the 64-bit mixing hash of the lattice key ints that the library and its checker share.
 *
 * Every function does the reference's IEEE double operations in the reference's order: explicit round-to-nearest intrinsics on
 * the device (never contracted to FMA), plain operators on the host (built with -ffp-contract=off).  Structurally-zero terms
 * are kept, so these forms match the reference for every control order at once.  The search kernel's own polynomial
 * (Axis<ORD>, mplb_device.cuh) and its filters drop those terms and are checked against the oracle instead.
 *
 * Plain C++ with no CUDA-only construct outside `#ifdef __CUDA_ARCH__`: the LPA* core that includes it is also compiled for
 * the host by the test suite (tests/cpp/lpa_emul.cpp).  Map helpers take any map description with `dim`, `nd[3]`, `origin[3]`
 * and `res` members.
 */
#ifndef MPLB_REF_H
#define MPLB_REF_H
#include <math.h>

#if defined(__CUDACC__)
#define MPLB_HD __host__ __device__ __forceinline__
#define MPLB_HDN __host__ __device__
#else
#define MPLB_HD inline
#define MPLB_HDN inline
#endif

namespace mplb_ref {

/* ------------------------------------------------------------------ IEEE operations without contraction */
#ifdef __CUDA_ARCH__
MPLB_HD double dadd(double a, double b) { return __dadd_rn(a, b); }
MPLB_HD double dsub(double a, double b) { return __dsub_rn(a, b); }
MPLB_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
MPLB_HD double ddiv(double a, double b) { return __ddiv_rn(a, b); }
MPLB_HD double dsqrt(double a) { return __dsqrt_rn(a); }
#else
MPLB_HD double dadd(double a, double b) { return a + b; }
MPLB_HD double dsub(double a, double b) { return a - b; }
MPLB_HD double dmul(double a, double b) { return a * b; }
MPLB_HD double ddiv(double a, double b) { return a / b; }
MPLB_HD double dsqrt(double a) { return sqrt(a); }
#endif
/* std::round (half away from zero), exact: x - trunc(x) is exactly representable */
MPLB_HD double round_haz(double x) {
  double r = trunc(x);
  if (fabs(dsub(x, r)) >= 0.5) r = dadd(r, copysign(1.0, x));
  return r;
}
/* (int)std::round(x) */
MPLB_HD int round_int(double x) {
#ifdef __CUDA_ARCH__
  return __double2int_rz(round_haz(x));
#else
  return (int)round_haz(x);
#endif
}
MPLB_HD double dmin(double a, double b) { return b < a ? b : a; } /* std::min */
MPLB_HD double dmax(double a, double b) { return a < b ? b : a; } /* std::max */
MPLB_HD double power(double t, int n) { /* mt:197-203 */
  double tn = 1;
  while (n > 0) { tn = dmul(tn, t); n--; }
  return tn;
}
MPLB_HD double normalize_angle(double a) { /* mt:15-19 */
  while (a > 3.141592653589793) a = dsub(a, 6.283185307179586);
  while (a < -3.141592653589793) a = dadd(a, 6.283185307179586);
  return a;
}
/* v.normalized().dot(Vec2f(cos yaw, sin yaw)) (pr:520, em:125): Eigen normalized() = v / sqrt(squaredNorm); cs, sn are the
 * correctly rounded cos / sin of the yaw (mplb_trig.cuh).  sqrt is IEEE-rounded in both builds. */
MPLB_HD double heading_dot(double vx, double vy, double cs, double sn) {
  const double z = dadd(dmul(vx, vx), dmul(vy, vy));
  double nx = vx, ny = vy;
  if (z > 0.0) { const double q = sqrt(z); nx = ddiv(vx, q); ny = ddiv(vy, q); }
  return dadd(dmul(nx, cs), dmul(ny, sn));
}

/* ------------------------------------------------------------------ Primitive1D (pr:21-198): c[0..5] = c0 .. c5 */
struct Prim1 { double c[6]; };
MPLB_HD double pr_p(const Prim1 &q, double t) { /* pr:128-131 */
  const double *c = q.c;
  double s = dmul(ddiv(c[0], 120), power(t, 5));
  s = dadd(s, dmul(ddiv(c[1], 24), power(t, 4)));
  s = dadd(s, dmul(ddiv(c[2], 6), power(t, 3)));
  s = dadd(s, dmul(dmul(ddiv(c[3], 2), t), t));
  s = dadd(s, dmul(c[4], t));
  return dadd(s, c[5]);
}
MPLB_HD double pr_v(const Prim1 &q, double t) { /* pr:134-137 */
  const double *c = q.c;
  double s = dmul(ddiv(c[0], 24), power(t, 4));
  s = dadd(s, dmul(ddiv(c[1], 6), power(t, 3)));
  s = dadd(s, dmul(dmul(ddiv(c[2], 2), t), t));
  s = dadd(s, dmul(c[3], t));
  return dadd(s, c[4]);
}
MPLB_HD double pr_a(const Prim1 &q, double t) { /* pr:140-142 */
  const double *c = q.c;
  double s = dmul(ddiv(c[0], 6), power(t, 3));
  s = dadd(s, dmul(dmul(ddiv(c[1], 2), t), t));
  s = dadd(s, dmul(c[2], t));
  return dadd(s, c[3]);
}
MPLB_HD double pr_j(const Prim1 &q, double t) { /* pr:145 */
  const double *c = q.c;
  return dadd(dadd(dmul(dmul(ddiv(c[0], 2), t), t), dmul(c[1], t)), c[2]);
}
/* solve(0, 0, c, d, e) of mt:117-131 (a = b = 0 for every control-built primitive: c0 = 0, pr:35-52); roots in the
 * order quad() returns them; returns the count */
MPLB_HD int solve_low(double c, double d, double e, double *r) {
  if (c != 0) { /* quad, mt:22-33 */
    const double p = dsub(dmul(d, d), dmul(dmul(4, c), e));
    if (p < 0) return 0;
    const double sq = dsqrt(p);
    r[0] = ddiv(dsub(-d, sq), dmul(2, c));
    r[1] = ddiv(dadd(-d, sq), dmul(2, c));
    return 2;
  } else if (d != 0) {
    r[0] = ddiv(-e, d);
    return 1;
  }
  return 0;
}
/* max over [0, T] of |derivative| (which = 1 vel, 2 acc, 3 jrk): end points and the interior extrema (pr:353-394 with
 * extrema_* pr:152-193) */
MPLB_HD double pr_max(const Prim1 &q, double T, int which) {
  const double *c = q.c;
  double r[2] = {0, 0};
  int nr = 0;
  double m;
  if (which == 1) { nr = solve_low(ddiv(c[1], 2), c[2], c[3], r); m = dmax(fabs(pr_v(q, 0)), fabs(pr_v(q, T))); }
  else if (which == 2) { nr = solve_low(0, c[1], c[2], r); m = dmax(fabs(pr_a(q, 0)), fabs(pr_a(q, T))); } /* solve(0,0,c0/2,c1,c2) */
  else { nr = 0; m = dmax(fabs(pr_j(q, 0)), fabs(pr_j(q, T))); } /* extrema_j needs c0 != 0 */
  for (int i = 0; i < nr; i++) { /* extrema_*: keep roots in (0, T), stop at the first root >= T */
    const double it = r[i];
    if (it > 0 && it < T) {
      const double x = fabs(which == 1 ? pr_v(q, it) : pr_a(q, it));
      m = x > m ? x : m;
    } else if (it >= T) break;
  }
  return m;
}
MPLB_HD double pr_J(const Prim1 &q, double t, int control) { /* pr:92-122 */
  const double *c = q.c;
  const int cc = control & 15;
  if (cc == 1) {
    double s = dmul(ddiv(dmul(c[0], c[0]), 5184), power(t, 9));
    s = dadd(s, dmul(ddiv(dmul(c[0], c[1]), 576), power(t, 8)));
    s = dadd(s, dmul(dadd(ddiv(dmul(c[1], c[1]), 252), ddiv(dmul(c[0], c[2]), 168)), power(t, 7)));
    s = dadd(s, dmul(dadd(ddiv(dmul(c[0], c[3]), 72), ddiv(dmul(c[1], c[2]), 36)), power(t, 6)));
    s = dadd(s, dmul(dadd(dadd(ddiv(dmul(c[2], c[2]), 20), ddiv(dmul(c[0], c[4]), 60)), ddiv(dmul(c[1], c[3]), 15)), power(t, 5)));
    s = dadd(s, dmul(dadd(ddiv(dmul(c[2], c[3]), 4), ddiv(dmul(c[1], c[4]), 12)), power(t, 4)));
    s = dadd(s, dmul(dadd(ddiv(dmul(c[3], c[3]), 3), ddiv(dmul(c[2], c[4]), 3)), power(t, 3)));
    s = dadd(s, dmul(dmul(dmul(c[3], c[4]), t), t));
    return dadd(s, dmul(dmul(c[4], c[4]), t));
  } else if (cc == 3) {
    double s = dmul(ddiv(dmul(c[0], c[0]), 252), power(t, 7));
    s = dadd(s, dmul(ddiv(dmul(c[0], c[1]), 36), power(t, 6)));
    s = dadd(s, dmul(dadd(ddiv(dmul(c[1], c[1]), 20), ddiv(dmul(c[0], c[2]), 15)), power(t, 5)));
    s = dadd(s, dmul(dadd(ddiv(dmul(c[0], c[3]), 12), ddiv(dmul(c[1], c[2]), 4)), power(t, 4)));
    s = dadd(s, dmul(dadd(ddiv(dmul(c[2], c[2]), 3), ddiv(dmul(c[1], c[3]), 3)), power(t, 3)));
    s = dadd(s, dmul(dmul(dmul(c[2], c[3]), t), t));
    return dadd(s, dmul(dmul(c[3], c[3]), t));
  } else if (cc == 7) {
    double s = dmul(ddiv(dmul(c[0], c[0]), 20), power(t, 5));
    s = dadd(s, dmul(ddiv(dmul(c[0], c[1]), 4), power(t, 4)));
    s = dadd(s, dmul(ddiv(dadd(dmul(c[1], c[1]), dmul(c[0], c[2])), 3), power(t, 3)));
    s = dadd(s, dmul(dmul(dmul(c[1], c[2]), t), t));
    return dadd(s, dmul(dmul(c[2], c[2]), t));
  } else if (cc == 15) {
    double s = dmul(ddiv(dmul(c[0], c[0]), 3), power(t, 3));
    s = dadd(s, dmul(dmul(dmul(c[0], c[1]), t), t));
    return dadd(s, dmul(dmul(c[1], c[1]), t));
  }
  return 0;
}

/* ------------------------------------------------------------------ Primitive (pr:205-431) without yaw */
struct Prim { Prim1 ax[3]; };
/* from a state row st (pos3 vel3 acc3 jrk3) and a control u, control order ord = 1 .. 4 (pr:35-52, 220-256) */
MPLB_HD void prim_build(int dim, int ord, const double *st, const double *u, Prim &pr) {
  for (int i = 0; i < dim; i++) {
    double *k = pr.ax[i].c;
    k[0] = k[1] = k[2] = k[3] = k[4] = k[5] = 0;
    if (ord == 4) { k[1] = u[i]; k[2] = st[9 + i]; k[3] = st[6 + i]; k[4] = st[3 + i]; k[5] = st[i]; }
    else if (ord == 3) { k[2] = u[i]; k[3] = st[6 + i]; k[4] = st[3 + i]; k[5] = st[i]; }
    else if (ord == 2) { k[3] = u[i]; k[4] = st[3 + i]; k[5] = st[i]; }
    else { k[4] = u[i]; k[5] = st[i]; }
  }
}
/* pr:321-331 into a 13-double state row; the yaw entry stays 0 */
MPLB_HD void prim_eval(int dim, const Prim &pr, double t, double *st) {
  for (int k = 0; k < 13; k++) st[k] = 0;
  for (int k = 0; k < dim; k++) {
    st[k] = pr_p(pr.ax[k], t);
    st[3 + k] = pr_v(pr.ax[k], t);
    st[6 + k] = pr_a(pr.ax[k], t);
    st[9 + k] = pr_j(pr.ax[k], t);
  }
}
MPLB_HD bool validate_xxx(int dim, const Prim &pr, double T, double mx, int which) { /* pr:483-496 */
  if (mx <= 0) return true;
  for (int i = 0; i < dim; i++)
    if (pr_max(pr.ax[i], T, which) > mx) return false;
  return true;
}
MPLB_HD bool validate_primitive(int dim, int ord, const Prim &pr, double T, double v_max, double a_max, double j_max) { /* pr:449-475 */
  if (ord == 2) return validate_xxx(dim, pr, T, v_max, 1);
  if (ord == 3) return validate_xxx(dim, pr, T, v_max, 1) && validate_xxx(dim, pr, T, a_max, 2);
  if (ord == 4) return validate_xxx(dim, pr, T, v_max, 1) && validate_xxx(dim, pr, T, a_max, 2) && validate_xxx(dim, pr, T, j_max, 3);
  return true;
}
MPLB_HD double prim_J(int dim, const Prim &pr, double T, int control) { /* pr:403-407 */
  double j = 0;
  for (int k = 0; k < dim; k++) j = dadd(j, pr_J(pr.ax[k], T, control));
  return j;
}
MPLB_HD double prim_max_v(int dim, const Prim &pr, double T) { /* the largest max_vel over the axes (em:91-94) */
  double mv = 0;
  for (int i = 0; i < dim; i++) {
    const double x = pr_max(pr.ax[i], T, 1);
    if (x > mv) mv = x;
  }
  return mv;
}

/* ------------------------------------------------------------------ MapUtil (map_util.h) */
MPLB_HD int float_to_cell(double pt, double origin, double res) { /* mu:103-108 on one axis: round((pt - origin)/res - 0.5) */
  return round_int(dsub(ddiv(dsub(pt, origin), res), 0.5));
}
template <class M>
MPLB_HD void float_to_int(const M &m, const double *pt, int *pn) { /* mu:103-108 */
  pn[0] = pn[1] = pn[2] = 0;
  for (int i = 0; i < m.dim; i++) pn[i] = float_to_cell(pt[i], m.origin[i], m.res);
}
template <class M>
MPLB_HD bool outside(const M &m, const int *pn) { /* mu:51-55 */
  for (int i = 0; i < m.dim; i++) if (pn[i] < 0 || pn[i] >= m.nd[i]) return true;
  return false;
}
template <class M>
MPLB_HD int cell_index(const M &m, const int *pn) { /* mu:33-41, int arithmetic like the reference (no bounds check) */
  return m.dim == 2 ? pn[0] + m.nd[0] * pn[1] : pn[0] + m.nd[0] * pn[1] + m.nd[0] * m.nd[1] * pn[2];
}
/* rayTrace (mu:117-134) from p1 to p2: ray_span writes diff = p2 - p1 and returns q / 0.8 (q = the largest |diff| / res over
 * the axes); ray_setup returns max_diff = (int)(q / 0.8) (points n = 1 .. max_diff - 1 are traced) and writes s = 1 / max_diff.
 * The reference takes std::max over the axes starting from 0; fmax is the same for these non-negative values and also skips a
 * NaN.  The cast is undefined unless q / 0.8 < 2^31, which a caller taking endpoints from outside checks with ray_span. */
MPLB_HD double ray_span(int dim, double res, const double *p1, const double *p2, double *diff) {
  double q = 0;
  for (int i = 0; i < dim; i++) {
    diff[i] = dsub(p2[i], p1[i]);
    q = fmax(q, fabs(ddiv(diff[i], res)));
  }
  return ddiv(q, 0.8);
}
MPLB_HD int ray_setup(int dim, double res, const double *p1, const double *p2, double *diff, double *s) {
  const int max_diff = (int)ray_span(dim, res, p1, p2, diff);
  *s = ddiv(1.0, (double)max_diff);
  return max_diff;
}
/* point n on one axis: pt1 + step * n with step = diff * s (mu:121,126) */
MPLB_HD double ray_point(double p1, double diff, double s, int n) { return dadd(p1, dmul(dmul(diff, s), (double)n)); }

/* ------------------------------------------------------------------ VoxelGrid (planning_ros_utils voxel_grid.cpp, vg) */
/* floatToInt (vg:201-203) on one axis: ((pt - origin_d_) / res_).cast<int>(), the float res_ widened to double and the
 * quotient TRUNCATED toward zero (not MapUtil's rounding).  Returns false where cast<int> is undefined (a NaN quotient or
 * one beyond int32); the grid treats such a point as outside. */
MPLB_HD bool vg_float_to_cell(double pt, double origin_d, float res, int *n) {
  const double q = ddiv(dsub(pt, origin_d), (double)res);
  if (!(q > -2147483649.0 && q < 2147483648.0)) return false;
#ifdef __CUDA_ARCH__
  *n = __double2int_rz(q);
#else
  *n = (int)q;
#endif
  return true;
}
/* intToFloat (vg:205-207) on one axis: (n + 0.5) * res_ + origin_d_ in that order */
MPLB_HD double vg_cell_to_float(int n, double origin_d, float res) {
  return dadd(dmul(dadd((double)n, 0.5), (double)res), origin_d);
}

/* ------------------------------------------------------------------ lattice key hash (library and checker definition) */
MPLB_HD unsigned long long khash_init() { return 0x243F6A8885A308D3ull; }
MPLB_HD unsigned long long khash_step(unsigned long long h, int v) {
  h ^= (unsigned long long)(unsigned int)v;
  h *= 0x9E3779B97F4A7C15ull;
  h ^= h >> 32;
  return h;
}
MPLB_HD unsigned long long khash_final(unsigned long long h) {
  h ^= h >> 30; h *= 0xBF58476D1CE4E5B9ull;
  h ^= h >> 27; h *= 0x94D049BB133111EBull;
  h ^= h >> 31;
  return h;
}
MPLB_HD unsigned long long key_hash(const int *k, int n) {
  unsigned long long h = khash_init();
  for (int i = 0; i < n; i++) h = khash_step(h, k[i]);
  return khash_final(h);
}

}  // namespace mplb_ref
#endif
